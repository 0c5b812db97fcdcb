"""On-GPU numerics + speed checks for the sm_90a kernel library.

usage: python scripts/gpu_check.py <section> [...]   sections: gemm gemm_bench misc attn all
Each section prints PASS/FAIL lines; exit code is non-zero on any FAIL.
"""
import sys
import time

import torch

from alpa_b200 import ops
_C = ops.native_module()

torch.manual_seed(0)
dev = "cuda"
FAILS = []


def check(name, got, ref, atol, rtol):
    got = got.float()
    ref = ref.float()
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = (err > tol).sum().item()
    ok = bad == 0 and torch.isfinite(got).all().item()
    print(f"{'PASS' if ok else 'FAIL'} {name}: max_abs_err={err.max().item():.4g} "
          f"ref_max={ref.abs().max().item():.4g} bad={bad}/{err.numel()}", flush=True)
    if not ok:
        FAILS.append(name)
    return ok


def timeit(fn, iters=20, warmup=5, flush=None):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        s = torch.cuda.Event(enable_timing=True)
        e = torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def sec_gemm():
    shapes = [(128, 256, 64), (128, 128, 128), (256, 512, 256), (1000, 520, 264), (4096, 2048, 2048),
              (384, 8, 64), (136, 2048, 72)]
    for (M, N, K) in shapes:
        for ta in (False, True):
            for tb in (False, True):
                a = torch.randn((K, M) if ta else (M, K), device=dev, dtype=torch.bfloat16)
                b = torch.randn((K, N) if tb else (N, K), device=dev, dtype=torch.bfloat16)
                A = a.float().t() if ta else a.float()
                B = b.float() if tb else b.float().t()
                ref = A @ B
                try:
                    out = _C.gemm(a, b, ta, tb)
                    torch.cuda.synchronize()
                    check(f"gemm M{M} N{N} K{K} ta={int(ta)} tb={int(tb)}", out, ref, 0.05 * K ** 0.5, 2e-2)
                except Exception as ex:  # noqa
                    print(f"FAIL gemm M{M} N{N} K{K} ta={int(ta)} tb={int(tb)}: {ex}")
                    FAILS.append("gemm-exc")
                    return
    # both tile widths explicitly
    for bn in (128, 256):
        a = torch.randn(512, 320, device=dev, dtype=torch.bfloat16)
        b = torch.randn(768, 320, device=dev, dtype=torch.bfloat16)
        out = _C.gemm(a, b, False, False, block_n=bn)
        check(f"gemm block_n={bn}", out, a.float() @ b.float().t(), 1.0, 2e-2)
    # batched
    a = torch.randn(6, 200, 128, device=dev, dtype=torch.bfloat16)
    b = torch.randn(6, 264, 128, device=dev, dtype=torch.bfloat16)
    out = _C.gemm(a, b, False, False)
    check("gemm batched NT", out, torch.bmm(a.float(), b.float().transpose(1, 2)), 0.6, 2e-2)
    b2 = torch.randn(6, 128, 264, device=dev, dtype=torch.bfloat16)
    out = _C.gemm(a, b2, False, True)
    check("gemm batched NN", out, torch.bmm(a.float(), b2.float()), 0.6, 2e-2)
    # epilogues
    M, N, K = 512, 1024, 256
    a = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
    w = torch.randn(N, K, device=dev, dtype=torch.bfloat16) * 0.1
    bias = torch.randn(N, device=dev, dtype=torch.bfloat16)
    res = torch.randn(M, N, device=dev, dtype=torch.bfloat16)
    z = a.float() @ w.float().t() + bias.float()
    out = _C.gemm(a, w, False, False, bias=bias)
    check("epi bias", out, z, 0.05, 2e-2)
    aux = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    out = _C.gemm(a, w, False, False, bias=bias, aux_out=aux, act=1)
    check("epi gelu", out, torch.nn.functional.gelu(z), 0.05, 2e-2)
    check("epi gelu aux", aux, z, 0.05, 2e-2)
    out = _C.gemm(a, w, False, False, bias=bias, act=2)
    check("epi relu", out, torch.relu(z), 0.05, 2e-2)
    out = _C.gemm(a, w, False, False, bias=bias, residual=res)
    check("epi residual", out, z + res.float(), 0.06, 2e-2)
    zz = torch.randn(M, N, device=dev, dtype=torch.bfloat16)
    zf = zz.float().requires_grad_(True)
    torch.nn.functional.gelu(zf).backward(torch.ones_like(zf))
    out = _C.gemm(a, w, False, False, aux_in=zz, act=3)
    check("epi dgelu", out, (a.float() @ w.float().t()) * zf.grad, 0.05, 2e-2)
    acc = torch.randn(M, N, device=dev, dtype=torch.float32)
    acc0 = acc.clone()
    _C.gemm(a, w, False, False, out=acc, accumulate=True)
    check("epi fp32 accumulate", acc, acc0 + a.float() @ w.float().t(), 0.05, 1e-2)
    out = _C.gemm(a, w, False, False, out_fp32=True, alpha=0.5)
    check("epi fp32 alpha", out, 0.5 * (a.float() @ w.float().t()), 0.05, 1e-2)
    # strided views (sharded slices)
    big = torch.randn(M, 2 * K, device=dev, dtype=torch.bfloat16)
    out = _C.gemm(big[:, K:], w, False, False)
    check("gemm strided A", out, big[:, K:].float() @ w.float().t(), 0.05, 2e-2)


def sec_gemm_bench():
    """The 15 GEMMs of one GPT-1.3B training step on one GPU (16 x 1024 tokens, H = 2048, 4H = 8192, V = 51200), with
    the operand majors, tile width and epilogues the step runs them with: the forward linears add the bias, fc1 also
    applies GELU and saves the pre-activation (aux_out), and the fc2 dgrad applies dGELU from it (aux_in).  The
    residual epilogue is not on this list: on one GPU the step adds the residual gradient in a separate kernel
    (ALPA_B200_FUSE_DGRAD_ADD is off by default).  M = 16384 makes A larger than the 50 MB L2, as in the step.
    cuBLAS runs the same product without the epilogue."""
    flush = torch.empty(256 * 1024 * 1024, device=dev, dtype=torch.uint8)
    T, H, I, V = 16384, 2048, 8192, 51200
    NONE, BIAS, GELU, DGELU = "", "bias", "bias+gelu+aux_out", "dgelu"
    shapes = []  # (name, M, N, K, trans_a, trans_b, epilogue)
    for name, n_in, n_out in (("qkv", H, 3 * H), ("proj", H, H), ("fc1", H, I), ("fc2", I, H), ("lm head", H, V)):
        shapes.append((f"{name} fwd", T, n_out, n_in, False, False, GELU if name == "fc1" else BIAS))
        shapes.append((f"{name} dgrad", T, n_in, n_out, False, True, DGELU if name == "fc2" else NONE))
        shapes.append((f"{name} wgrad", n_out, n_in, T, True, True, NONE))
    for name, M, N, K, ta, tb, epi in shapes:
        a = torch.randn((K, M) if ta else (M, K), device=dev, dtype=torch.bfloat16)
        b = torch.randn((K, N) if tb else (N, K), device=dev, dtype=torch.bfloat16) * K ** -0.5
        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        kw = {}
        if epi in (BIAS, GELU):
            kw["bias"] = torch.randn(N, device=dev, dtype=torch.bfloat16)
        if epi == GELU:
            kw.update(aux_out=torch.empty(M, N, device=dev, dtype=torch.bfloat16), act=1)
        if epi == DGELU:
            kw.update(aux_in=torch.randn(M, N, device=dev, dtype=torch.bfloat16), act=3)
        A = a.t() if ta else a
        B = b if tb else b.t()
        ref_out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        t = timeit(lambda: _C.gemm(a, b, ta, tb, out=out, **kw), flush=flush)
        t2 = timeit(lambda: torch.matmul(A, B, out=ref_out), flush=flush)
        fl = 2 * M * N * K / 1e9
        print(f"BENCH gemm {name:12s} M={M:5d} N={N:5d} K={K:5d} {epi or '-':17s}: {t:.3f} ms {fl / t:6.1f} TFLOPS | "
              f"cublas {t2:.3f} ms {fl / t2:6.1f} TFLOPS", flush=True)
        ref = ref_out.float()
        if "bias" in kw:
            ref = ref + kw["bias"].float()
        if epi == GELU:
            ref = torch.nn.functional.gelu(ref)
        if epi == DGELU:
            z = kw["aux_in"].float().requires_grad_(True)
            torch.nn.functional.gelu(z).backward(torch.ones_like(z))
            ref = ref * z.grad
        check(f"bench-correct {name}", out, ref, 0.05, 3e-2)
        del a, b, out, ref_out, ref, kw


def sec_misc():
    # LayerNorm
    for rows, H in [(64, 256), (4096, 2048), (1000, 5120), (33, 1024)]:
        x = torch.randn(rows, H, device=dev, dtype=torch.bfloat16)
        r = torch.randn(rows, H, device=dev, dtype=torch.bfloat16)
        g = torch.randn(H, device=dev, dtype=torch.bfloat16)
        b = torch.randn(H, device=dev, dtype=torch.bfloat16)
        y, mean, rstd, _ = _C.layernorm_fwd(x, None, g, b, 1e-5, False)
        ref = torch.nn.functional.layer_norm(x.float(), (H,), g.float(), b.float(), 1e-5)
        check(f"ln fwd {rows}x{H}", y, ref, 0.03, 2e-2)
        y2, mean2, rstd2, s2 = _C.layernorm_fwd(x, r, g, b, 1e-5, True)
        s_ref = (x.float() + r.float()).bfloat16()
        check(f"ln fwd+res sum {rows}x{H}", s2, s_ref, 0.02, 1e-2)
        check(f"ln fwd+res {rows}x{H}", y2,
              torch.nn.functional.layer_norm(s_ref.float(), (H,), g.float(), b.float(), 1e-5), 0.03, 2e-2)
        dy = torch.randn(rows, H, device=dev, dtype=torch.bfloat16)
        xf = x.float().requires_grad_(True)
        gf = g.float().requires_grad_(True)
        bf = b.float().requires_grad_(True)
        torch.nn.functional.layer_norm(xf, (H,), gf, bf, 1e-5).backward(dy.float())
        dg = torch.zeros(H, device=dev)
        db = torch.zeros(H, device=dev)
        dx = _C.layernorm_bwd(dy, x, g, mean, rstd, None, dg, db)
        check(f"ln bwd dx {rows}x{H}", dx, xf.grad, 0.05, 3e-2)
        check(f"ln bwd dgamma {rows}x{H}", dg, gf.grad, 0.02 * rows ** 0.5 + 0.05, 2e-2)
        check(f"ln bwd dbeta {rows}x{H}", db, bf.grad, 0.02 * rows ** 0.5 + 0.05, 2e-2)
        dx2 = _C.layernorm_bwd(dy, x, g, mean, rstd, r, dg, db)
        check(f"ln bwd dx+dres {rows}x{H}", dx2, xf.grad + r.float(), 0.06, 3e-2)
    # cross entropy
    T, V = 512, 51200
    logits = torch.randn(T, V, device=dev, dtype=torch.bfloat16) * 2
    labels = torch.randint(0, V, (T,), device=dev)
    stats = _C.ce_stats(logits, labels, 0)
    lf = logits.float()
    check("ce max", stats[:, 0], lf.max(dim=1).values, 1e-3, 1e-3)
    check("ce sumexp", stats[:, 1], torch.exp(lf - lf.max(dim=1, keepdim=True).values).sum(1), 1e-2, 1e-3)
    check("ce tgt", stats[:, 2], lf.gather(1, labels[:, None])[:, 0], 1e-3, 1e-3)
    loss = torch.log(stats[:, 1]) + stats[:, 0] - stats[:, 2]
    ref_loss = torch.nn.functional.cross_entropy(lf, labels, reduction="none")
    check("ce loss", loss, ref_loss, 1e-2, 1e-3)
    lfg = lf.clone().requires_grad_(True)
    torch.nn.functional.cross_entropy(lfg, labels, reduction="mean").backward()
    g = logits.clone()
    _C.ce_grad_(g, labels, stats[:, :2].contiguous(), torch.full((T,), 1.0 / T, device=dev), 0)
    check("ce grad", g, lfg.grad, 2e-5, 2e-2)
    # vocab-parallel halves
    half = V // 2
    s0 = _C.ce_stats(logits[:, :half], labels, 0)
    s1 = _C.ce_stats(logits[:, half:], labels, half)
    gmax = torch.maximum(s0[:, 0], s1[:, 0])
    gsum = s0[:, 1] * torch.exp(s0[:, 0] - gmax) + s1[:, 1] * torch.exp(s1[:, 0] - gmax)
    check("ce vocab-parallel loss", torch.log(gsum) + gmax - (s0[:, 2] + s1[:, 2]), ref_loss, 1e-2, 1e-3)
    # embedding
    Vv, H = 1000, 512
    wte = torch.randn(Vv, H, device=dev, dtype=torch.bfloat16)
    wpe = torch.randn(128, H, device=dev, dtype=torch.bfloat16)
    ids = torch.randint(0, Vv, (4, 128), device=dev)
    pos = torch.arange(128, device=dev).repeat(4, 1).contiguous()
    e = _C.embedding_fwd(ids, pos, wte, wpe, 0)
    check("embedding fwd", e, (wte[ids].float() + wpe[pos].float()), 0.03, 1e-2)
    e2 = _C.embedding_fwd(ids, None, wte[500:].contiguous(), None, 500)
    ref2 = torch.where((ids >= 500)[..., None], wte[ids].float(), torch.zeros(1, device=dev))
    check("embedding fwd vocab-parallel", e2, ref2, 1e-3, 1e-3)
    dy = torch.randn(4, 128, H, device=dev, dtype=torch.bfloat16)
    dt = torch.zeros(Vv, H, device=dev)
    _C.embedding_bwd_(ids, dy, dt, 0)
    ref = torch.zeros(Vv, H, device=dev).index_add_(0, ids.flatten(), dy.float().view(-1, H))
    check("embedding bwd", dt, ref, 1e-3, 1e-3)
    # colsum
    x = torch.randn(3000, 768, device=dev, dtype=torch.bfloat16)
    o = torch.zeros(768, device=dev)
    _C.colsum_(x, o)
    check("colsum", o, x.float().sum(0), 0.05, 1e-3)
    # adamw
    ps = [torch.randn(n, device=dev) for n in (1000, 65536 * 2 + 3, 7)]
    gs = [torch.randn_like(p) for p in ps]
    gs[1] = gs[1].bfloat16()
    ms = [torch.zeros_like(p) for p in ps]
    vs = [torch.zeros_like(p) for p in ps]
    pb = [torch.empty_like(p, dtype=torch.bfloat16) for p in ps]
    ref_p = [p.clone().requires_grad_(True) for p in ps]
    opt = torch.optim.AdamW([{"params": ref_p[:2], "weight_decay": 0.01}, {"params": ref_p[2:], "weight_decay": 0.0}],
                            lr=1e-2, betas=(0.9, 0.999), eps=1e-8)
    tt, cc, *_host = _C.adam_build_tables(gs, ps, ms, vs, pb, [0.01, 0.01, 0.0])
    for step in (1, 2, 3):
        for rp, g in zip(ref_p, gs):
            rp.grad = g.float().clone()
        opt.step()
        _C.adamw_step(tt, cc, 1e-2, 0.9, 0.999, 1e-8, step, 1.0, None)
    for i in range(3):
        check(f"adamw master[{i}]", ps[i], ref_p[i].detach(), 1e-5, 1e-4)
        check(f"adamw bf16[{i}]", pb[i], ref_p[i].detach(), 1e-2, 1e-2)
    ss = _C.grad_sumsq(tt, cc)
    check("grad sumsq", ss[0], sum((g.float() ** 2).sum() for g in gs), 1.0, 1e-3)
    # bandwidth numbers
    flush = torch.empty(256 * 1024 * 1024, device=dev, dtype=torch.uint8)
    rows, H = 16384, 2048
    x = torch.randn(rows, H, device=dev, dtype=torch.bfloat16)
    g = torch.ones(H, device=dev, dtype=torch.bfloat16)
    b = torch.zeros(H, device=dev, dtype=torch.bfloat16)
    t = timeit(lambda: _C.layernorm_fwd(x, None, g, b, 1e-5, False), flush=flush)
    print(f"BENCH ln fwd {rows}x{H}: {t * 1e3:.1f} us  {2 * rows * H * 2 / t / 1e6:.0f} GB/s")
    n = 256 * 1024 * 1024
    p = torch.zeros(n, device=dev); gg = torch.zeros(n, device=dev)
    m = torch.zeros(n, device=dev); v = torch.zeros(n, device=dev)
    pbf = torch.zeros(n, device=dev, dtype=torch.bfloat16)
    tt, cc, *_host = _C.adam_build_tables([gg], [p], [m], [v], [pbf], [0.01])
    t = timeit(lambda: _C.adamw_step(tt, cc, 1e-3, 0.9, 0.999, 1e-8, 1, 1.0, None))
    print(f"BENCH adamw {n} elems: {t:.3f} ms  {n * (16 + 12 + 2) / t / 1e6:.0f} GB/s")


def sec_attn():
    from scripts import gpu_check_attn
    gpu_check_attn.run(check, timeit, FAILS)


def sec_moe():
    """MoE routing / dispatch / combine / batched GEMM: native vs the PyTorch reference path of the same op."""
    from alpa_b200.global_env import global_config
    torch.manual_seed(3)

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
        check(f"moe route expert {tag}", ex, ex_r, 0, 0)
        check(f"moe route slot {tag}", sl, sl_r, 0, 0)
        x = torch.randn(G, S, M, device=dev, dtype=torch.bfloat16)
        w = torch.rand(G, S, 2, device=dev, dtype=torch.bfloat16)
        for wt in (None, w):
            d, d_r = both(lambda: ops.moe_dispatch(x, ex_r, sl_r, wt, E, C))
            check(f"moe dispatch w={wt is not None} {tag}", d, d_r, 1e-2, 1e-2)
            eo = torch.randn(E, G * C, M, device=dev, dtype=torch.bfloat16)
            o, o_r = both(lambda: ops.moe_combine(eo, ex_r, sl_r, wt))
            check(f"moe combine w={wt is not None} {tag}", o, o_r, 2e-2, 2e-2)
        dw, dw_r = both(lambda: ops.moe_combine_wgrad(x, eo, ex_r, sl_r))
        check(f"moe combine_wgrad {tag}", dw, dw_r, 0.5, 2e-2)
    for (B, Mm, N, K) in [(4, 256, 128, 64), (8, 1024, 2048, 1024), (3, 136, 72, 200)]:
        for ta in (False, True):
            for tb in (False, True):
                a = torch.randn((B, K, Mm) if ta else (B, Mm, K), device=dev, dtype=torch.bfloat16)
                b = torch.randn((B, K, N) if tb else (B, N, K), device=dev, dtype=torch.bfloat16)
                c = ops.bmm(a, b, ta, tb)
                ref = torch.matmul(a.float().transpose(1, 2) if ta else a.float(), b.float() if tb else b.float().transpose(1, 2))
                check(f"bmm B{B} M{Mm} N{N} K{K} ta={int(ta)} tb={int(tb)}", c, ref, 0.3, 2e-2)
    # speed: the MoE-2.4B layer shapes (E=16, M=1024, H=4096... per-GPU tokens 8x1024)
    flush = torch.empty(256 * 1024 * 1024, device=dev, dtype=torch.uint8)
    G, S, E, M, H = 4, 2048, 16, 1024, 4096
    C = 2 * S // E
    gates = torch.softmax(torch.randn(G, S, E, device=dev), -1)
    ex, sl = ops.moe_top2_route(gates, C)
    x = torch.randn(G, S, M, device=dev, dtype=torch.bfloat16)
    w = torch.rand(G, S, 2, device=dev, dtype=torch.bfloat16)
    t = timeit(lambda: ops.moe_top2_route(gates, C), flush=flush)
    print(f"BENCH moe route G{G} S{S} E{E}: {t * 1e3:.1f} us")
    t = timeit(lambda: ops.moe_dispatch(x, ex, sl, None, E, C), flush=flush)
    print(f"BENCH moe dispatch: {t * 1e3:.1f} us  {(x.numel() * 2 * 3 + E * G * C * M * 2) / t / 1e6:.0f} GB/s (incl. zero fill)")
    d = ops.moe_dispatch(x, ex, sl, None, E, C)
    t = timeit(lambda: ops.moe_combine(d, ex, sl, w), flush=flush)
    print(f"BENCH moe combine: {t * 1e3:.1f} us  {(x.numel() * 2 * 3) / t / 1e6:.0f} GB/s")
    wi = torch.randn(E, M, H, device=dev, dtype=torch.bfloat16)
    t = timeit(lambda: ops.bmm(d, wi, False, True), flush=flush)
    print(f"BENCH moe expert bmm [{E},{G * C},{M}]x[{E},{M},{H}]: {t * 1e3:.1f} us {2.0 * E * G * C * M * H / t / 1e9:.0f} TFLOPS")


def _bench_note(line):
    """Timing lines of the GPU checks; also appended to $ALPA_B200_BENCH_NOTES when set (pytest drops stdout)."""
    import os
    print("BENCH " + line, flush=True)
    path = os.environ.get("ALPA_B200_BENCH_NOTES")
    if path:
        with open(path, "a") as f:
            f.write(line + "\n")


def sec_gemv():
    """Decode GEMV (fp8 / bf16 weights, fused bias / activation / residual) vs an fp32 reference."""
    torch.manual_seed(3)
    from alpa_b200.ops import primitives as P
    for (M, N, K) in [(1, 2560, 2560), (4, 7680, 2560), (8, 2560, 10240), (3, 1000, 512), (1, 50272, 2560), (2, 24, 64)]:
        x = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
        w = torch.randn(N, K, device=dev, dtype=torch.float32) * 0.05
        b = torch.randn(N, device=dev, dtype=torch.bfloat16)
        r = torch.randn(M, N, device=dev, dtype=torch.bfloat16)
        scale = (w.abs().amax(1).clamp(min=1e-8) / 448.0)
        w8 = (w / scale[:, None]).to(torch.float8_e4m3fn)
        # fp8 weights: activations are quantised per token to e4m3 inside the kernel (like the prefill fp8 GEMM);
        # the reference uses the same quantised operands, so the comparison tests the kernel, not the rounding
        sx = x.float().abs().amax(1, keepdim=True).clamp(min=1e-8) / 448.0
        xq = (x.float() / sx).to(torch.float8_e4m3fn).float() * sx
        for act in ("none", "gelu"):
            y = _C.gemv_decode(x, w8, scale, b, r, {"none": 0, "gelu": 1}[act])
            ref = torch.nn.functional.linear(xq, w8.float() * scale[:, None], b.float())
            ref = (torch.nn.functional.gelu(ref) if act == "gelu" else ref) + r.float()
            check(f"gemv fp8 {act} M{M} N{N} K{K}", y, ref, 0.06, 2e-2)
        ref_unq = torch.nn.functional.linear(x.float(), w8.float() * scale[:, None], b.float()) + r.float()
        y = _C.gemv_decode(x, w8, scale, b, r, 0)
        err = (y.float() - ref_unq).abs().max().item() / ref_unq.abs().max().item()
        print(f"INFO gemv fp8 M{M} N{N} K{K}: activation-quantisation error {err:.4f} of max |y|", flush=True)
        wb = w.bfloat16()
        y = _C.gemv_decode(x, wb, None, None, None, 0)
        check(f"gemv bf16 M{M} N{N} K{K}", y, x.float() @ wb.float().t(), 0.06, 2e-2)
    # bandwidth: OPT-2.7B fc1 at batch 1 (26 MB of e4m3 weights).  Ten different weight matrices back to back inside
    # one timed region: 260 MB > L2, and the launch latency of a single tiny kernel does not pollute the number
    x = torch.randn(1, 2560, device=dev, dtype=torch.bfloat16)
    w8s = [(torch.randn(10240, 2560, device=dev) * 0.05).to(torch.float8_e4m3fn) for _ in range(10)]
    w8 = w8s[0]
    sc = torch.ones(10240, device=dev)
    flush = None

    def many(fn):
        def run():
            for w_ in w8s:
                fn(w_)
        return run
    t = timeit(many(lambda w_: _C.gemv_decode(x, w_, sc, None, None, 0))) / len(w8s)
    print(f"BENCH gemv fp8 M1 N10240 K2560: {t * 1e3:.1f} us  {w8.numel() / t / 1e9:.2f} TB/s", flush=True)
    y2 = P.linear_decode(x, w8, sc)
    check("linear_decode primitive", y2, _C.gemv_decode(x, w8, sc, None, None, 0), 1e-6, 0)
    # layer norm fused into the prologue
    for (M, N, K) in [(1, 7680, 2560), (8, 1024, 2560), (2, 512, 8192), (3, 264, 1088)]:
        x = torch.randn(M, K, device=dev, dtype=torch.bfloat16) * 3 + 0.5
        g = (1 + 0.1 * torch.randn(K, device=dev)).bfloat16()
        be = (0.1 * torch.randn(K, device=dev)).bfloat16()
        wb = (torch.randn(N, K, device=dev) * 0.05).bfloat16()
        b = torch.randn(N, device=dev, dtype=torch.bfloat16)
        y = _C.gemv_decode(x, wb, None, b, None, 0, g, be, 1e-5)
        xn = torch.nn.functional.layer_norm(x.float(), (K,), g.float(), be.float(), 1e-5).bfloat16().float()
        check(f"gemv LN prologue M{M} N{N} K{K}", y, xn @ wb.float().t() + b.float(), 0.08, 2e-2)
        sw = wb.float().abs().amax(1).clamp(min=1e-8) / 448.0
        wq = (wb.float() / sw[:, None]).to(torch.float8_e4m3fn)
        y8 = _C.gemv_decode(x, wq, sw, b, None, 0, g, be, 1e-5)
        sxn = xn.abs().amax(1, keepdim=True).clamp(min=1e-8) / 448.0
        xnq = (xn / sxn).to(torch.float8_e4m3fn).float() * sxn
        check(f"gemv fp8 LN prologue M{M} N{N} K{K}", y8, xnq @ (wq.float() * sw[:, None]).t() + b.float(), 0.08, 2e-2)
    x = torch.randn(1, 2560, device=dev, dtype=torch.bfloat16)
    g = torch.ones(2560, device=dev, dtype=torch.bfloat16)
    be = torch.zeros(2560, device=dev, dtype=torch.bfloat16)
    t2 = timeit(many(lambda w_: _C.gemv_decode(x, w_, sc, None, None, 0, g, be, 1e-5))) / len(w8s)
    print(f"BENCH gemv fp8+LN M1 N10240 K2560: {t2 * 1e3:.1f} us", flush=True)
    _bench_note(f"gemv fp8 M1 N10240 K2560: {t * 1e3:.1f} us ({w8.numel() / t / 1e9:.2f} TB/s); with LN prologue {t2 * 1e3:.1f} us")
    # decode attention with fused cache append vs the reference (append, then masked attention)
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
        check(f"decode_attention B{B} h{h} D{D} n{n}", o, ref, 0.03, 2e-2)
        check(f"decode_attention cache append B{B} n{n}", torch.stack([kc, vc]), torch.stack([kc2, vc2]), 1e-6, 0)
    B, h, D, S_max, n = 1, 32, 80, 1024, 545
    qkv = torch.randn(B, 1, h, 3, D, device=dev, dtype=torch.bfloat16)
    kc = torch.randn(B, S_max, h, D, device=dev, dtype=torch.bfloat16)
    vc = torch.randn(B, S_max, h, D, device=dev, dtype=torch.bfloat16)
    kv = torch.tensor([n], device=dev, dtype=torch.int32)
    caches = [(torch.randn_like(kc), torch.randn_like(vc)) for _ in range(16)]          # 16 x 2 x 5.2 MB

    def attn_all():
        for kc_, vc_ in caches:
            P.decode_attention(qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2], kc_, vc_, kv, D ** -0.5)
    t3 = timeit(attn_all) / len(caches)
    _bench_note(f"decode_attention B1 h32 D80 ctx545: {t3 * 1e3:.1f} us")


def sec_fp8():
    """fp8 (e4m3) serving GEMM: per-token activation scales x per-channel weight scales, vs fp32 of the same
    quantised operands (exactness of the kernel) and vs the unquantised product (quantisation error)."""
    torch.manual_seed(5)
    for (M, N, K, act, use_bias) in [(128, 256, 256, "none", True), (4, 7680, 2560, "none", True),
                                     (1000, 2560, 10240, "none", False), (2048, 10240, 2560, "relu", True),
                                     (130, 72, 528, "gelu", True)]:
        x = (torch.randn(M, K, device=dev) * 0.7).to(torch.bfloat16)
        w = torch.randn(N, K, device=dev) * 0.05
        b = (torch.randn(N, device=dev) * 0.1).to(torch.bfloat16) if use_bias else None
        sw = (w.abs().amax(1).clamp(min=1e-8) / 448.0).float()
        wq = (w / sw[:, None]).to(torch.float8_e4m3fn)
        y = ops.linear_fp8(x, wq, sw, b, act)
        # reference on the quantised operands
        sx = (x.float().abs().amax(1).clamp(min=1e-8) / 448.0)
        xq = (x.float() / sx[:, None]).to(torch.float8_e4m3fn).float()
        ref = (xq @ wq.float().t()) * sx[:, None] * sw[None, :]
        if b is not None:
            ref = ref + b.float()
        if act == "relu":
            ref = torch.relu(ref)
        elif act == "gelu":
            ref = torch.nn.functional.gelu(ref)
        check(f"fp8 gemm M{M} N{N} K{K} {act}", y, ref, 2e-2 * (K ** 0.5) * 0.05 + 2e-2, 2e-2)
        full = x.float() @ w.t()
        rel = ((y.float() - (torch.relu(full + (b.float() if b is not None else 0)) if act == "relu" else
                             (torch.nn.functional.gelu(full + (b.float() if b is not None else 0)) if act == "gelu"
                              else full + (b.float() if b is not None else 0)))).norm() / full.norm()).item()
        print(f"INFO fp8 quantisation rel err M{M} N{N} K{K}: {rel:.4f}")
    flush = torch.empty(256 * 1024 * 1024, device=dev, dtype=torch.uint8)
    for (M, N, K) in [(2048, 7680, 2560), (2048, 10240, 2560), (2048, 2560, 10240), (8192, 8192, 8192), (8, 10240, 2560)]:
        x = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
        w = torch.randn(N, K, device=dev) * 0.05
        sw = (w.abs().amax(1) / 448.0).float()
        wq = (w / sw[:, None]).to(torch.float8_e4m3fn)
        wb = w.to(torch.bfloat16)
        t8 = timeit(lambda: ops.linear_fp8(x, wq, sw, None, "none"), flush=flush)
        t16 = timeit(lambda: ops.linear(x, wb, None), flush=flush)
        print(f"BENCH linear M{M} N{N} K{K}: fp8 (incl. activation quantisation) {t8 * 1e3:.1f} us "
              f"{2.0 * M * N * K / t8 / 1e9:.0f} TFLOPS | bf16 {t16 * 1e3:.1f} us {2.0 * M * N * K / t16 / 1e9:.0f} TFLOPS")


def sec_ragged():
    """ragged 1-D attention over a slot-addressed KV cache vs the fp32 reference (OPT-2.7B/TP1 head shapes)."""
    from alpa_b200 import ops
    from alpa_b200.ops import primitives as P
    torch.manual_seed(0)
    dev = "cuda"
    for (h, D, lens, new) in [(4, 64, [37, 1, 300, 129], [5, 1, 1, 129]), (32, 80, [512, 77, 2048, 1000], [1, 1, 1, 64]),
                              (8, 128, [16, 4000], [16, 1])]:
        slots = sum(lens) + 64
        kc = torch.randn(slots + 1, h, D, device=dev, dtype=torch.bfloat16)
        vc = torch.randn(slots + 1, h, D, device=dev, dtype=torch.bfloat16)
        starts, s = [], 7
        for n in lens:
            starts.append(s)
            s += n + 3
        seq_start, ctx_len = [], []
        for st, n, k in zip(starts, lens, new):            # the last `k` tokens of each sequence are queries
            for j in range(n - k, n):
                seq_start.append(st)
                ctx_len.append(j + 1)
        seq_start += [0, 0]
        ctx_len += [0, 0]                                   # padding tokens
        T = len(seq_start)
        q = torch.randn(T, h, 3, D, device=dev, dtype=torch.bfloat16)[:, :, 0]          # strided view like qkv
        ss = torch.tensor(seq_start, dtype=torch.int32, device=dev)
        cl = torch.tensor(ctx_len, dtype=torch.int32, device=dev)
        mc = max(lens)
        for alibi in (None, torch.linspace(0.01, 0.2, h, device=dev)):
            got = ops.ragged_attention(q, kc, vc, ss, cl, D ** -0.5, mc, alibi)
            old = P.global_config.use_native_kernels
            P.global_config.use_native_kernels = False
            try:
                ref = ops.ragged_attention(q.float(), kc.float(), vc.float(), ss, cl, D ** -0.5, mc, alibi)
            finally:
                P.global_config.use_native_kernels = old
            check(f"ragged_attention h{h} D{D} T{T} alibi={alibi is not None}", got, ref, 2e-2, 2e-2)
        t = timeit(lambda: ops.ragged_attention(q, kc, vc, ss, cl, D ** -0.5, mc, None))
        kv_bytes = sum(c * h * D * 2 * 2 for c in ctx_len)
        print(f"BENCH ragged_attention h{h} D{D} T{T}: {t * 1e3:.1f} us, {kv_bytes / t / 1e6:.0f} GB/s of K/V streamed")


if __name__ == "__main__":
    secs = sys.argv[1:] or ["all"]
    print(torch.cuda.get_device_name(0), torch.__version__, flush=True)
    t0 = time.time()
    for s in secs:
        if s in ("gemm", "all"):
            sec_gemm()
        if s in ("gemm_bench", "all"):
            sec_gemm_bench()
        if s in ("misc", "all"):
            sec_misc()
        if s in ("attn",):
            sec_attn()
        if s in ("moe",):
            sec_moe()
        if s in ("fp8",):
            sec_fp8()
        if s in ("ragged",):
            sec_ragged()
    print(f"done in {time.time() - t0:.1f}s; FAILS={FAILS}")
    sys.exit(1 if FAILS else 0)
