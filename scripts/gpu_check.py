"""Kernel timings on the GPU: one section per kernel group, each printing `BENCH` lines (CUDA events, median of 20
calls after 5 warm-ups).  The kernels' numerics are checked by the GPU tests under tests/.

usage: python scripts/gpu_check.py [section ...]
  sections: gemm_bench gemm_sweep misc attn attn_gqa moe fp8 gemv ragged llama llama_step llama_decode kv_fp8
            ragged_paged paged_prefill
            (default: all)
gemm_bench also checks the outputs it times; the exit code is non-zero if one is wrong.
"""
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from alpa_b200 import ops  # noqa: E402
from alpa_b200.ops import primitives as P  # noqa: E402
from alpa_b200.util import benchmark_cuda_events  # noqa: E402
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


def median_ms(fn, flush=False):
    """Median time of fn() in ms over 20 calls after 5 warm-ups; the L2 is flushed before each call if `flush`."""
    ts = np.sort(benchmark_cuda_events(fn, warmup=5, repeat=20, flush_l2=flush))
    return ts[len(ts) // 2] * 1e3


def sec_gemm_bench():
    """The 15 GEMMs of one GPT-1.3B training step on one GPU (16 x 1024 tokens, H = 2048, 4H = 8192, V = 51200), with
    the operand majors, tile width and epilogues the step runs them with: the forward linears add the bias, fc1 also
    applies GELU and saves the pre-activation (aux_out), and the fc2 dgrad applies dGELU from it (aux_in).  The
    residual epilogue is not on this list: on one GPU the step adds the residual gradient in a separate kernel
    (ALPA_B200_FUSE_DGRAD_ADD is off by default).  M = 16384 makes A larger than the 50 MB L2, as in the step.
    cuBLAS runs the same product without the epilogue.  No test runs these shapes, so the timed outputs are checked."""
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
        t = median_ms(lambda: _C.gemm(a, b, ta, tb, out=out, **kw), flush=True)
        t2 = median_ms(lambda: torch.matmul(A, B, out=ref_out), flush=True)
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


def sec_gemm_sweep():
    """Per-tile cost model of the bf16 GEMM: M = 16384, N = 6144 (qkv fwd) with 128 x 256 tiles, K from 512 to 8192,
    for each epilogue the training step uses.  The persistent kernel runs ceil(tiles / #SMs) rounds of one tile per
    SM, so time / rounds = slope * K + intercept.  The slope is the mainloop's rate (printed as TFLOPS over all SMs);
    the intercept is what every tile costs besides its K loop: pipeline fill, epilogue and stores.  Each epilogue runs
    with the operand majors the step uses it with: dGELU in the dgrad layout (B stored [K, N]), the others forward."""
    M, N = 16384, 6144
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rounds = math.ceil(math.ceil(M / 128) * math.ceil(N / 256) / sms)
    Ks = (512, 1024, 2048, 4096, 8192)
    bias = torch.randn(N, device=dev, dtype=torch.bfloat16)
    aux = torch.randn(M, N, device=dev, dtype=torch.bfloat16)
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    epilogues = (("-", False, {}), ("bias", False, {"bias": bias}),
                 ("bias+gelu+aux_out", False, {"bias": bias, "aux_out": aux, "act": 1}),
                 ("dgelu", True, {"aux_in": aux, "act": 3}))
    for name, tb, kw in epilogues:
        per_round = []
        for K in Ks:
            a = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
            b = torch.randn((K, N) if tb else (N, K), device=dev, dtype=torch.bfloat16) * K ** -0.5
            t = median_ms(lambda: _C.gemm(a, b, False, tb, out=out, block_n=256, **kw), flush=True)
            per_round.append(t * 1e3 / rounds)
            print(f"BENCH gemm_sweep {name:17s} M={M} N={N} K={K:5d}: {t:.3f} ms "
                  f"{2 * M * N * K / t / 1e9:6.1f} TFLOPS  {per_round[-1]:.2f} us/round", flush=True)
            del a, b
        slope, icpt = np.polyfit(np.array(Ks, dtype=np.float64), np.array(per_round), 1)
        print(f"FIT gemm_sweep {name:17s}: mainloop {2 * 128 * 256 * sms / slope / 1e6:.0f} TFLOPS, "
              f"intercept {icpt:.1f} us/tile ({rounds} rounds of {sms} tiles)", flush=True)


def sec_misc():
    """LayerNorm forward and AdamW bandwidth."""
    rows, H = 16384, 2048
    x = torch.randn(rows, H, device=dev, dtype=torch.bfloat16)
    g = torch.ones(H, device=dev, dtype=torch.bfloat16)
    b = torch.zeros(H, device=dev, dtype=torch.bfloat16)
    t = median_ms(lambda: _C.layernorm_fwd(x, None, g, b, 1e-5, False), flush=True)
    print(f"BENCH ln fwd {rows}x{H}: {t * 1e3:.1f} us  {2 * rows * H * 2 / t / 1e6:.0f} GB/s")
    n = 256 * 1024 * 1024
    p = torch.zeros(n, device=dev); gg = torch.zeros(n, device=dev)
    m = torch.zeros(n, device=dev); v = torch.zeros(n, device=dev)
    pbf = torch.zeros(n, device=dev, dtype=torch.bfloat16)
    tt, cc, *_host = _C.adam_build_tables([gg], [p], [m], [v], [pbf], [0.01])
    t = median_ms(lambda: _C.adamw_step(tt, cc, 1e-3, 0.9, 0.999, 1e-8, 1, 1.0, None))
    print(f"BENCH adamw {n} elems: {t:.3f} ms  {n * (16 + 12 + 2) / t / 1e6:.0f} GB/s")


def sec_attn():
    """Attention forward (against SDPA) and backward at the GPT-1.3B (32 heads x 64) and 15B (40 x 128) head shapes."""
    for (B, H, S, D, causal) in [(8, 32, 1024, 64, False), (8, 32, 1024, 64, True), (8, 40, 1024, 128, False),
                                 (2, 32, 4096, 64, False)]:
        qkv = torch.randn(B, S, 3, H, D, device=dev, dtype=torch.bfloat16)
        q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
        scale = 1.0 / math.sqrt(D)
        t = median_ms(lambda: _C.attention_fwd(q, k, v, scale, causal), flush=True)
        fl = 4 * B * H * S * S * D * (0.5 if causal else 1.0)
        print(f"BENCH attn fwd B{B} H{H} S{S} D{D} causal={int(causal)}: {t:.3f} ms {fl / t / 1e9:.1f} TFLOPS", flush=True)
        qq, kk, vv = (x.transpose(1, 2) for x in (q, k, v))
        t2 = median_ms(lambda: torch.nn.functional.scaled_dot_product_attention(qq, kk, vv, is_causal=causal), flush=True)
        print(f"BENCH sdpa(lib) fwd same: {t2:.3f} ms {fl / t2 / 1e9:.1f} TFLOPS", flush=True)
        o, lse = _C.attention_fwd(q, k, v, scale, causal)
        do = torch.randn_like(o)
        t = median_ms(lambda: _C.attention_bwd(do, q, k, v, o, lse, scale, causal), flush=True)
        print(f"BENCH attn bwd B{B} H{H} S{S} D{D} causal={int(causal)}: {t:.3f} ms {2.5 * fl / t / 1e9:.1f} TFLOPS", flush=True)


def sec_attn_gqa():
    """Grouped-query attention against what a user does without it: the multi-head kernel on K/V expanded with
    repeat_interleave (the expansion itself not timed), whose backward needs the group sum of dK / dV on top, and
    torch's SDPA with enable_gqa.  Shapes: Llama-3-8B-like on one GPU; one GPU of an 8-way tensor-parallel 70B-like
    model (one K/V head: the dK / dV group split); multi-query attention."""
    for (B, S, Hq, Hkv, D, causal) in [(4, 2048, 32, 8, 128, True), (1, 4096, 8, 1, 128, True),
                                       (8, 1024, 32, 1, 64, False)]:
        G = Hq // Hkv
        qkv = torch.randn(B, S, Hkv, G + 2, D, device=dev, dtype=torch.bfloat16)
        q, k, v = qkv[:, :, :, :G], qkv[:, :, :, G], qkv[:, :, :, G + 1]
        scale = 1.0 / math.sqrt(D)
        fl = 4 * B * Hq * S * S * D * (0.5 if causal else 1.0)
        tag = f"B{B} S{S} Hq{Hq} Hkv{Hkv} D{D} causal={int(causal)}"
        splits = _C.attention_bwd_splits(q, k, v)

        def row(name, t, flops):
            print(f"BENCH attn_gqa {tag} {name}: {t:.3f} ms {flops / t / 1e9:.1f} TFLOPS", flush=True)

        row("gqa fwd", median_ms(lambda: _C.attention_fwd(q, k, v, scale, causal), flush=True), fl)
        o, lse = _C.attention_fwd(q, k, v, scale, causal)
        do = torch.randn_like(o)
        row(f"gqa bwd (dK/dV group split {splits})",
            median_ms(lambda: _C.attention_bwd(do, q, k, v, o, lse, scale, causal), flush=True), 2.5 * fl)
        qe = q.reshape(B, S, Hq, D)
        ke, ve = (x.repeat_interleave(G, dim=2) for x in (k, v))
        row("mha fwd on expanded K/V", median_ms(lambda: _C.attention_fwd(qe, ke, ve, scale, causal), flush=True), fl)
        oe, lsee = _C.attention_fwd(qe, ke, ve, scale, causal)
        doe = do.reshape(B, S, Hq, D)

        def mha_bwd():
            dq, dk, dv = _C.attention_bwd(doe, qe, ke, ve, oe, lsee, scale, causal)
            return dk.view(B, S, Hkv, G, D).sum(3), dv.view(B, S, Hkv, G, D).sum(3)
        row("mha bwd on expanded K/V + group sum", median_ms(mha_bwd, flush=True), 2.5 * fl)
        qt, kt, vt = qe.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
        row("sdpa(lib) enable_gqa fwd", median_ms(lambda: torch.nn.functional.scaled_dot_product_attention(
            qt, kt, vt, is_causal=causal, scale=scale, enable_gqa=True), flush=True), fl)


def sec_moe():
    """MoE routing, dispatch, combine and expert GEMM at the MoE-2.4B layer shapes (E = 16, M = 1024, H = 4096)."""
    G, S, E, M, H = 4, 2048, 16, 1024, 4096
    C = 2 * S // E
    gates = torch.softmax(torch.randn(G, S, E, device=dev), -1)
    ex, sl = ops.moe_top2_route(gates, C)
    x = torch.randn(G, S, M, device=dev, dtype=torch.bfloat16)
    w = torch.rand(G, S, 2, device=dev, dtype=torch.bfloat16)
    t = median_ms(lambda: ops.moe_top2_route(gates, C), flush=True)
    print(f"BENCH moe route G{G} S{S} E{E}: {t * 1e3:.1f} us")
    t = median_ms(lambda: ops.moe_dispatch(x, ex, sl, None, E, C), flush=True)
    print(f"BENCH moe dispatch: {t * 1e3:.1f} us  {(x.numel() * 2 * 3 + E * G * C * M * 2) / t / 1e6:.0f} GB/s (incl. zero fill)")
    d = ops.moe_dispatch(x, ex, sl, None, E, C)
    t = median_ms(lambda: ops.moe_combine(d, ex, sl, w), flush=True)
    print(f"BENCH moe combine: {t * 1e3:.1f} us  {(x.numel() * 2 * 3) / t / 1e6:.0f} GB/s")
    wi = torch.randn(E, M, H, device=dev, dtype=torch.bfloat16)
    t = median_ms(lambda: ops.bmm(d, wi, False, True), flush=True)
    print(f"BENCH moe expert bmm [{E},{G * C},{M}]x[{E},{M},{H}]: {t * 1e3:.1f} us {2.0 * E * G * C * M * H / t / 1e9:.0f} TFLOPS")


def sec_fp8():
    """fp8 (e4m3, per-token x per-channel scales) serving GEMMs against the bf16 GEMM, and the MXFP8 GEMM at 8192^3."""
    for (M, N, K) in [(2048, 7680, 2560), (2048, 10240, 2560), (2048, 2560, 10240), (8192, 8192, 8192), (8, 10240, 2560)]:
        x = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
        w = torch.randn(N, K, device=dev) * 0.05
        sw = (w.abs().amax(1) / 448.0).float()
        wq = (w / sw[:, None]).to(torch.float8_e4m3fn)
        wb = w.to(torch.bfloat16)
        t8 = median_ms(lambda: ops.linear_fp8(x, wq, sw, None, "none"), flush=True)
        t16 = median_ms(lambda: ops.linear(x, wb, None), flush=True)
        print(f"BENCH linear M{M} N{N} K{K}: fp8 (incl. activation quantisation) {t8 * 1e3:.1f} us "
              f"{2.0 * M * N * K / t8 / 1e9:.0f} TFLOPS | bf16 {t16 * 1e3:.1f} us {2.0 * M * N * K / t16 / 1e9:.0f} TFLOPS")
    M = N = K = 8192
    q, sf = _C.quantize_mxfp8(torch.randn(M, K, device=dev, dtype=torch.bfloat16))
    wq, wsf = _C.quantize_mxfp8(torch.randn(N, K, device=dev, dtype=torch.bfloat16))
    t = median_ms(lambda: _C.gemm_mxfp8_q(q, sf, wq, wsf, None, 0), flush=True)
    print(f"BENCH mxfp8 gemm 8192^3 (operands pre-quantised): {t:.3f} ms {2 * M * N * K / t / 1e9:.0f} TFLOPS", flush=True)


def sec_gemv():
    """Decode GEMV (OPT-2.7B fc1 at batch 1, 26 MB of e4m3 weights), without and with the LayerNorm prologue, and
    decode attention with the cache append (OPT-2.7B heads, 545 tokens of context)."""
    # ten different weight matrices back to back inside one timed region: 260 MB > L2, and the launch latency of a
    # single tiny kernel does not pollute the number
    x = torch.randn(1, 2560, device=dev, dtype=torch.bfloat16)
    w8s = [(torch.randn(10240, 2560, device=dev) * 0.05).to(torch.float8_e4m3fn) for _ in range(10)]
    sc = torch.ones(10240, device=dev)

    def many(fn):
        def run():
            for w_ in w8s:
                fn(w_)
        return run
    t = median_ms(many(lambda w_: _C.gemv_decode(x, w_, sc, None, None, 0))) / len(w8s)
    print(f"BENCH gemv fp8 M1 N10240 K2560: {t * 1e3:.1f} us  {w8s[0].numel() / t / 1e9:.2f} TB/s", flush=True)
    g = torch.ones(2560, device=dev, dtype=torch.bfloat16)
    be = torch.zeros(2560, device=dev, dtype=torch.bfloat16)
    t = median_ms(many(lambda w_: _C.gemv_decode(x, w_, sc, None, None, 0, g, be, 1e-5))) / len(w8s)
    print(f"BENCH gemv fp8+LN M1 N10240 K2560: {t * 1e3:.1f} us", flush=True)
    B, h, D, S_max, n = 1, 32, 80, 1024, 545
    qkv = torch.randn(B, 1, h, 3, D, device=dev, dtype=torch.bfloat16)
    kv = torch.tensor([n], device=dev, dtype=torch.int32)
    caches = [(torch.randn(B, S_max, h, D, device=dev, dtype=torch.bfloat16),
               torch.randn(B, S_max, h, D, device=dev, dtype=torch.bfloat16)) for _ in range(16)]   # 16 x 2 x 5.2 MB

    def attn_all():
        for kc_, vc_ in caches:
            P.decode_attention(qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2], kc_, vc_, kv, D ** -0.5)
    t = median_ms(attn_all) / len(caches)
    print(f"BENCH decode_attention B{B} h{h} D{D} ctx{n}: {t * 1e3:.1f} us", flush=True)


def sec_ragged():
    """Ragged 1-D attention over a slot-addressed KV cache (OPT-2.7B/TP1 head shapes)."""
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
        t = median_ms(lambda: ops.ragged_attention(q, kc, vc, ss, cl, D ** -0.5, max(lens), None))
        kv_bytes = sum(c * h * D * 2 * 2 for c in ctx_len)
        print(f"BENCH ragged_attention h{h} D{D} T{T}: {t * 1e3:.1f} us, {kv_bytes / t / 1e6:.0f} GB/s of K/V streamed")


# The 1.3B-sized Llama-style config of the llama sections: 16 x 1024 tokens, H = 2048, 32 query heads, 8 K/V heads,
# D = 64, I = 5504 (GPT-1.3B's width and depth with Llama's block).
LLAMA_B, LLAMA_S, LLAMA_H, LLAMA_HQ, LLAMA_HKV, LLAMA_I = 16, 1024, 2048, 32, 8, 5504


def sec_llama():
    """RMSNorm, rotary and SwiGLU at the Llama-style step shapes, L2 flushed, against the LayerNorm kernel and the eager
    PyTorch compositions a user would otherwise run (F.rms_norm; HF's cos / sin and apply_rotary_pos_emb on separate
    q / k; F.silu(g) * u on the interleaved pairs).  GB/s counts the bytes each op must move at least."""
    from transformers.models.llama.modeling_llama import apply_rotary_pos_emb
    F = torch.nn.functional
    bf = torch.bfloat16
    T, H, Hq, Hkv, I = LLAMA_B * LLAMA_S, LLAMA_H, LLAMA_HQ, LLAMA_HKV, LLAMA_I
    D, G = H // Hq, Hq // Hkv

    def row(name, t, nbytes):
        print(f"BENCH llama {name}: {t * 1e3:.1f} us  {nbytes / t / 1e6:.0f} GB/s", flush=True)

    x = torch.randn(T, H, device=dev, dtype=bf)
    g = (1 + 0.1 * torch.randn(H, device=dev)).to(bf)
    b = torch.zeros(H, device=dev, dtype=bf)
    dy = torch.randn(T, H, device=dev, dtype=bf)
    row(f"rmsnorm fwd {T}x{H}", median_ms(lambda: _C.layernorm_fwd(x, None, g, None, 1e-5, False, rms=True),
                                          flush=True), 2 * T * H * 2)
    row(f"layernorm fwd {T}x{H}", median_ms(lambda: _C.layernorm_fwd(x, None, g, b, 1e-5, False), flush=True),
        2 * T * H * 2)
    row(f"F.rms_norm(lib) fwd {T}x{H}", median_ms(lambda: F.rms_norm(x, (H,), g, 1e-5), flush=True), 2 * T * H * 2)
    _, mean, rstd_ln, _ = _C.layernorm_fwd(x, None, g, b, 1e-5, False)
    _, _, rstd, _ = _C.layernorm_fwd(x, None, g, None, 1e-5, False, rms=True)
    dg, db = torch.zeros(H, device=dev), torch.zeros(H, device=dev)
    row(f"rmsnorm bwd {T}x{H}", median_ms(lambda: _C.layernorm_bwd(dy, x, g, None, rstd, None, dg, None, rms=True),
                                          flush=True), 3 * T * H * 2)
    row(f"layernorm bwd {T}x{H}", median_ms(lambda: _C.layernorm_bwd(dy, x, g, mean, rstd_ln, None, dg, db),
                                            flush=True), 3 * T * H * 2)
    xr, gr = x.clone().requires_grad_(), g.clone().requires_grad_()
    yr = F.rms_norm(xr, (H,), gr, 1e-5)
    row(f"F.rms_norm(lib) bwd {T}x{H}", median_ms(lambda: torch.autograd.grad(yr, (xr, gr), dy, retain_graph=True),
                                                  flush=True), 3 * T * H * 2)

    qkv = torch.randn(LLAMA_B, LLAMA_S, Hkv, G + 2, D, device=dev, dtype=bf)
    pos = torch.arange(LLAMA_S, device=dev).repeat(LLAMA_B, 1)
    nbytes = 2 * qkv.numel() * 2
    row(f"rotary fwd B{LLAMA_B} S{LLAMA_S} Hq{Hq} Hkv{Hkv} D{D}",
        median_ms(lambda: ops.rotary_packed(qkv, pos, 10000.0, False), flush=True), nbytes)
    inv = P._inv_freq(D, 10000.0, str(qkv.device))
    q = torch.randn(LLAMA_B, LLAMA_S, Hq, D, device=dev, dtype=bf).transpose(1, 2)   # HF's [B, heads, S, D] views
    k = torch.randn(LLAMA_B, LLAMA_S, Hkv, D, device=dev, dtype=bf).transpose(1, 2)

    def hf_rotary():
        freqs = (inv[None, :, None].expand(LLAMA_B, -1, 1) @ pos[:, None, :].float()).transpose(1, 2)
        emb = torch.cat((freqs, freqs), dim=-1)
        return apply_rotary_pos_emb(q, k, emb.cos().to(bf), emb.sin().to(bf))
    row("HF apply_rotary_pos_emb(lib) q+k incl. cos/sin", median_ms(hf_rotary, flush=True),
        2 * (q.numel() + k.numel()) * 2)

    gu = torch.randn(T, I, 2, device=dev, dtype=bf)
    dh = torch.randn(T, I, device=dev, dtype=bf)
    row(f"swiglu fwd {T}x{I}", median_ms(lambda: ops.swiglu(gu), flush=True), T * I * 6)
    row(f"F.silu(g)*u(lib) fwd {T}x{I}", median_ms(lambda: F.silu(gu[..., 0]) * gu[..., 1], flush=True), T * I * 6)
    row(f"swiglu bwd {T}x{I}", median_ms(lambda: ops.swiglu_bwd(dh, gu), flush=True), T * I * 10)
    gur = gu.clone().requires_grad_()
    hr = F.silu(gur[..., 0]) * gur[..., 1]
    row(f"F.silu(g)*u(lib) bwd {T}x{I}", median_ms(lambda: torch.autograd.grad(hr, gur, dh, retain_graph=True),
                                                   flush=True), T * I * 10)


def sec_llama_step():
    """One-GPU training of the 1.3B-sized Llama-style config through ShardParallel (fused AdamW on fp32 masters, as
    bench.py trains GPT-1.3B): ms per step from CUDA events, the RMSNorm (with its dgamma reduction) / rotary / SwiGLU
    kernels' share of one profiled step, and the library fallbacks (none expected)."""
    import alpa_b200 as alpa
    from alpa_b200.model.gpt_model import GPTConfig, GPTModel, gpt_lm_loss, num_params
    from alpa_b200.model.model_util import TrainState, adamw, functional_call, params_of
    alpa.init(cluster="local")
    cfg = GPTConfig(arch="llama", vocab_size=51200, hidden_size=LLAMA_H, num_hidden_layers=24,
                    num_attention_heads=LLAMA_HQ, num_key_value_heads=LLAMA_HKV, intermediate_size=LLAMA_I,
                    causal=True, layer_norm_eps=1e-5, dtype=torch.bfloat16)
    model = GPTModel(cfg, device=dev)
    state = TrainState.create(apply_fn=None, params=params_of(model), use_master_copy=True, tx=adamw(1e-4, fused=True))

    def train_step(state, batch):
        def loss_fn(p):
            return gpt_lm_loss(functional_call(model, p, (batch["input_ids"], batch["position_ids"])), batch["labels"])
        loss, grads = alpa.value_and_grad(loss_fn)(state.params)
        return state.apply_gradients(grads=grads), loss

    step = alpa.parallelize(train_step, method=alpa.ShardParallel(), donate_argnums=(0,))
    B, S = LLAMA_B, LLAMA_S
    batch = {"input_ids": torch.randint(1, cfg.vocab_size, (B, S), device=dev),
             "position_ids": torch.arange(S, device=dev).repeat(B, 1),
             "labels": torch.randint(1, cfg.vocab_size, (B, S), device=dev)}
    losses = []
    for _ in range(3):
        state, loss = step(state, batch)
    torch.cuda.synchronize()
    n = 10
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        state, loss = step(state, batch)
        losses.append(loss)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    print(f"BENCH llama_step {num_params(cfg) / 1e9:.2f}B params, B{B} S{S}: {ms:.1f} ms/step, "
          f"{B * S / ms * 1e3:.0f} tokens/s, losses {float(losses[0]._value):.4f} -> {float(losses[-1]._value):.4f}",
          flush=True)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        state, loss = step(state, batch)
        torch.cuda.synchronize()
    total, share = 0.0, {}
    for ev in prof.key_averages():
        t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        total += t
        name = ev.key
        # reduce_slots_kernel sums the RMSNorm backward's dgamma slots; its other users (bias gradients, grad-norm
        # clipping) do not run in this step, which is checked below
        kind = ("rotary" if "rotary_packed_kernel" in name else "swiglu" if "swiglu_" in name else
                "rmsnorm" if ("layernorm" in name and "true>" in name) or "reduce_slots_kernel" in name else None)
        if kind:
            share[kind] = share.get(kind, 0.0) + t
        if "colsum_kernel" in name or "sumsq_kernel" in name:
            FAILS.append(f"llama_step: {name} also uses reduce_slots_kernel; the RMSNorm share would include it")
    for kind, t in sorted(share.items()):
        print(f"BENCH llama_step kernel share {kind}: {t / 1e3:.2f} ms of {total / 1e3:.2f} ms GPU time "
              f"({100 * t / total:.1f} %)", flush=True)
    fb = P.library_fallbacks()
    print(f"llama_step library_fallbacks: {fb}", flush=True)
    if fb:
        FAILS.append("llama_step library fallbacks")
    alpa.shutdown()


def sec_llama_decode():
    """Grouped-query decode attention (fused rotary + cache append) at the Llama-3-8B shape (Hkv = 8, G = 4, D = 128),
    against the multi-head kernel on the cache expanded to 32 heads, which is what serving GQA took before.  Bytes are
    the K / V rows each kernel must read (2 * B * kv_len * heads * D * 2); the share is of 3.35 TB/s (H100 SXM data
    sheet), for the grouped kernel's bytes.  L2 flushed before each call."""
    Hkv, G, D, theta = 8, 4, 128, 500000.0
    scale = D ** -0.5
    print("llama_decode: B ctx | grouped us GB/s share | expanded-MHA us GB/s | speed-up", flush=True)
    for B in (1, 8, 32):
        for ctx in (1024, 4096, 16384):
            torch.manual_seed(0)
            qkv = torch.randn(B, 1, Hkv, G + 2, D, device="cuda", dtype=torch.bfloat16)
            kc = torch.randn(B, ctx, Hkv, D, device="cuda", dtype=torch.bfloat16)
            vc = torch.randn_like(kc)
            kv_len = torch.full((1,), ctx, dtype=torch.int32, device="cuda")
            pos = torch.full((B, 1), ctx - 1, dtype=torch.long, device="cuda")
            t_g = median_ms(lambda: ops.fast.decode_attention_gqa(qkv, kc, vc, kv_len, pos, scale, theta), flush=True)
            o_g = ops.fast.decode_attention_gqa(qkv, kc, vc, kv_len, pos, scale, theta)
            # the expanded multi-head form of the same step: rotated row, K / V repeated per query head
            rot = ops.rotary_packed(qkv, pos, theta, False)
            q = rot[:, :, :, :G].reshape(B, 1, Hkv * G, D)
            kn = rot[:, :, :, G:G + 1].expand(-1, -1, -1, G, -1).reshape(B, 1, Hkv * G, D).contiguous()
            vn = rot[:, :, :, G + 1:].expand(-1, -1, -1, G, -1).reshape(B, 1, Hkv * G, D).contiguous()
            ke = kc.repeat_interleave(G, 2)
            ve = vc.repeat_interleave(G, 2)
            del kc, vc
            t_e = median_ms(lambda: ops.fast.decode_attention(q, kn, vn, ke, ve, kv_len, scale), flush=True)
            o_e = ops.fast.decode_attention(q, kn, vn, ke, ve, kv_len, scale)
            check(f"llama_decode B={B} ctx={ctx} grouped vs expanded", o_g.float(), o_e.float(), 2e-2, 2e-2)
            nbytes = 2 * B * ctx * Hkv * D * 2
            gbs_g, gbs_e = nbytes / t_g / 1e6, G * nbytes / t_e / 1e6
            print(f"llama_decode: B={B:2d} ctx={ctx:5d} | {t_g * 1e3:8.1f} us {gbs_g:7.0f} GB/s "
                  f"{gbs_g / 3350:5.1%} | {t_e * 1e3:8.1f} us {gbs_e:7.0f} GB/s | {t_e / t_g:4.2f}x", flush=True)
            del ke, ve
            torch.cuda.empty_cache()


def sec_kv_fp8():
    """The grouped decode kernel over a bf16 and over an fp8 cache at the Llama-3-8B shape (Hkv = 8, G = 4, D = 128),
    timed alternately (bf16, fp8, bf16, fp8; the median of each kernel's two medians), L2 flushed before each call.
    Bytes are the cache bytes each kernel must read: per K / V row and head, D * 2 (bf16) or D + 4 (e4m3 + its fp32
    scale); the share is of 3.35 TB/s (H100 SXM data sheet).  The fp8 cache holds the bf16 cache's rows quantised by
    the store kernel; the two outputs are checked against each other."""
    Hkv, G, D, theta = 8, 4, 128, 500000.0
    scale = D ** -0.5
    print("kv_fp8: B ctx | bf16 us GB/s share | fp8 us GB/s share | fp8 speed-up", flush=True)
    for B in (1, 8, 32):
        for ctx in (1024, 4096, 16384):
            torch.manual_seed(0)
            qkv = torch.randn(B, 1, Hkv, G + 2, D, device="cuda", dtype=torch.bfloat16)
            kc = torch.randn(B, ctx, Hkv, D, device="cuda", dtype=torch.bfloat16)
            vc = torch.randn_like(kc)
            k8, v8 = ops.Fp8KV.zeros(kc.shape, "cuda"), ops.Fp8KV.zeros(kc.shape, "cuda")
            ops.kv_cache_store(kc, vc, k8, v8, 0)
            kv_len = torch.full((1,), ctx, dtype=torch.int32, device="cuda")
            pos = torch.full((B, 1), ctx - 1, dtype=torch.long, device="cuda")
            runs = {"bf16": lambda: ops.fast.decode_attention_gqa(qkv, kc, vc, kv_len, pos, scale, theta),
                    "fp8": lambda: ops.fast.decode_attention_gqa(qkv, k8, v8, kv_len, pos, scale, theta)}
            ts = {k: [] for k in runs}
            for _ in range(2):
                for k, fn in runs.items():
                    ts[k].append(median_ms(fn, flush=True))
            t = {k: float(np.median(v)) for k, v in ts.items()}
            check(f"kv_fp8 B={B} ctx={ctx} fp8 vs bf16 cache", runs["fp8"]().float(), runs["bf16"]().float(), 2e-2,
                  1e-1)
            rows = 2 * B * ctx * Hkv
            gbs = {"bf16": rows * D * 2 / t["bf16"] / 1e6, "fp8": rows * (D + 4) / t["fp8"] / 1e6}
            print(f"kv_fp8: B={B:2d} ctx={ctx:5d} | {t['bf16'] * 1e3:8.1f} us {gbs['bf16']:7.0f} GB/s "
                  f"{gbs['bf16'] / 3350:5.1%} | {t['fp8'] * 1e3:8.1f} us {gbs['fp8']:7.0f} GB/s {gbs['fp8'] / 3350:5.1%}"
                  f" | {t['bf16'] / t['fp8']:4.2f}x", flush=True)
            del kc, vc, k8, v8
            torch.cuda.empty_cache()


def _scatter_blocks(c, perm, bs):
    """A copy of slot-addressed cache c whose block perm[L] holds c's block L (the scratch row stays last)."""
    nblk = perm.numel()
    if isinstance(c, torch.Tensor):
        out = torch.empty_like(c)
        out[:nblk * bs].view(nblk, -1)[perm.long()] = c[:nblk * bs].view(nblk, -1)
        return out
    data = torch.empty_like(c.data.view(torch.uint8))
    data[:nblk * bs].view(nblk, -1)[perm.long()] = c.data.view(torch.uint8)[:nblk * bs].view(nblk, -1)
    scale = torch.empty_like(c.scale)
    H = scale.shape[0]
    scale[:, :nblk * bs].view(H, nblk, bs)[:, perm.long()] = c.scale[:, :nblk * bs].view(H, nblk, bs)
    return ops.Fp8KV(data.view(torch.float8_e4m3fn), scale)


def sec_ragged_paged():
    """The ragged kernel over a paged cache against the contiguous kernel on the same logical keys, at the Llama-3-8B
    attention shape (h = 32, Hkv = 8, D = 128): 64 and 256 decode tokens, each with its own sequence of 1024 / 4096 /
    16384 keys, and one 512-token prompt chunk at keys 3585..4096.  The contiguous cache gives sequence i rows
    [i * ctx, (i + 1) * ctx); the paged cache holds the same keys in blocks scattered by a random permutation, read
    through the matching table.  Timed alternately (contiguous, paged, twice; the median of each kernel's two
    medians), L2 flushed before each call.  Bytes are the K and V bytes of each token's keys, counted once per token
    (the 4 query heads of a group share them): per row and head D * 2 (bf16) or D + 4 (e4m3 and its fp32 scale).  The
    two outputs must be bitwise equal."""
    h, Hkv, D = 32, 8, 128
    scale = D ** -0.5
    print("ragged_paged: cache T ctx bs | contiguous us GB/s | paged us GB/s | paged / contiguous time", flush=True)
    cases = [(T, ctx, False) for T in (64, 256) for ctx in (1024, 4096, 16384)] + [(512, 4096, True)]
    for cache in ("bf16", "fp8"):
        for T, ctx, chunk in cases:
            torch.manual_seed(0)
            nseq = 1 if chunk else T
            slots = nseq * ctx
            q = torch.randn(T, h, D, device="cuda", dtype=torch.bfloat16)
            if cache == "bf16":
                kc = torch.randn(slots + 1, Hkv, D, device="cuda", dtype=torch.bfloat16)
                vc = torch.randn_like(kc)
            else:
                kc, vc = ops.Fp8KV.zeros((slots + 1, Hkv, D), "cuda"), ops.Fp8KV.zeros((slots + 1, Hkv, D), "cuda")
                for r0 in range(0, slots, 1 << 19):
                    n = min(1 << 19, slots - r0)
                    k = torch.randn(1, n, Hkv, D, device="cuda", dtype=torch.bfloat16)
                    ops.kv_cache_store(k, torch.randn_like(k), kc, vc, 0, torch.arange(r0, r0 + n, device="cuda"))
            if chunk:
                cl = torch.arange(ctx - T + 1, ctx + 1, dtype=torch.int32, device="cuda")
                seq = torch.zeros(T, dtype=torch.int32, device="cuda")
            else:
                cl = torch.full((T,), ctx, dtype=torch.int32, device="cuda")
                seq = torch.arange(T, dtype=torch.int32, device="cuda")
            row_bytes = Hkv * (D * 2 if cache == "bf16" else D + 4)
            nbytes = 2 * row_bytes * int(cl.sum())
            for bs in (16, 64):
                perm = torch.randperm(slots // bs, device="cuda").to(torch.int32)
                kp, vp = _scatter_blocks(kc, perm, bs), _scatter_blocks(vc, perm, bs)
                table = perm.view(nseq, ctx // bs)
                runs = {"contiguous": lambda: ops.fast.ragged_attention(q, kc, vc, seq * ctx, cl, scale, ctx),
                        "paged": lambda: ops.fast.ragged_attention(q, kp, vp, seq, cl, scale, ctx, None, table, bs)}
                check(f"ragged_paged {cache} T={T} ctx={ctx} bs={bs} paged == contiguous bitwise",
                      runs["paged"](), runs["contiguous"](), 0, 0)
                ts = {k: [] for k in runs}
                for _ in range(2):
                    for k, fn in runs.items():
                        ts[k].append(median_ms(fn, flush=True))
                t = {k: float(np.median(v)) for k, v in ts.items()}
                cols = " | ".join(f"{t[k] * 1e3:8.1f} us {nbytes / t[k] / 1e6:6.0f} GB/s" for k in runs)
                print(f"ragged_paged: {cache:4s} T={T:3d} ctx={ctx:5d}{' chunk' if chunk else '      '} bs={bs:2d} | "
                      f"{cols} | {t['paged'] / t['contiguous']:.3f}", flush=True)
                del kp, vp, runs
                torch.cuda.empty_cache()
            del kc, vc
            torch.cuda.empty_cache()


def sec_paged_prefill():
    """The paged prefill kernel (wgmma) against the paged ragged kernel (CUDA cores) on the same prompt chunks, at the
    Llama-3-8B attention shape (h = 32, Hkv = 8, D = 128): one 512-token chunk at keys 3585..4096, one 2048-token chunk
    after a 6144-token cached prefix, and a batch of four chunks of mixed lengths and prefixes; blocks of 16 and 64
    rows scattered by a random permutation.  Timed alternately (ragged, prefill, twice; the median of each kernel's two
    medians), L2 flushed before each call.  FLOPs are the causal ones: 4 * D * h per (query, visible key).  The share
    of peak is against the data sheet's 989 TFLOP/s dense bf16."""
    h, Hkv, D = 32, 8, 128
    scale = D ** -0.5
    print("paged_prefill: chunks bs | ragged us TFLOP/s | prefill us TFLOP/s % of 989 | ragged / prefill time",
          flush=True)
    cases = {"512@3584": [(3584, 512)], "2048@6144": [(6144, 2048)],
             "mixed": [(1024, 100), (4000, 300), (0, 64), (2000, 700)]}
    for name, chunks in cases.items():
        torch.manual_seed(0)
        for bs in (16, 64):
            nb = [-(-(p + n) // bs) for p, n in chunks]
            width = max(nb)
            nblk = sum(nb)
            perm = torch.randperm(nblk, device="cuda").to(torch.int32)
            table = torch.zeros(len(chunks), width, dtype=torch.int32, device="cuda")
            o = 0
            for i, n in enumerate(nb):
                table[i, :n] = perm[o:o + n]
                o += n
            kc = torch.randn(nblk * bs + 1, Hkv, D, device="cuda", dtype=torch.bfloat16)
            vc = torch.randn_like(kc)
            T = sum(n for _, n in chunks)
            q = torch.randn(T, h, D, device="cuda", dtype=torch.bfloat16)
            i32 = lambda x: torch.tensor(x, dtype=torch.int32, device="cuda")  # noqa: E731
            cs = i32([sum(n for _, n in chunks[:i]) for i in range(len(chunks))])
            cl, cp = i32([n for _, n in chunks]), i32([p for p, _ in chunks])
            seq = i32([i for i, (_, n) in enumerate(chunks) for _ in range(n)])
            ctx = i32([p + j + 1 for p, n in chunks for j in range(n)])
            mc = width * bs
            flops = 4 * D * h * int(ctx.sum())
            runs = {"ragged": lambda: ops.fast.ragged_attention(q, kc, vc, seq, ctx, scale, mc, None, table, bs),
                    "prefill": lambda: ops.fast.paged_prefill_attention(q, kc, vc, table, bs, cs, cl, cp, scale, mc)}
            check(f"paged_prefill {name} bs={bs} prefill ~ ragged", runs["prefill"](), runs["ragged"](), 2e-2, 2e-2)
            ts = {k: [] for k in runs}
            for _ in range(2):
                for k, fn in runs.items():
                    ts[k].append(median_ms(fn, flush=True))
            t = {k: float(np.median(v)) for k, v in ts.items()}
            tf = {k: flops / t[k] / 1e9 for k in runs}
            print(f"paged_prefill: {name:10s} bs={bs:2d} | {t['ragged'] * 1e3:9.1f} us {tf['ragged']:6.1f} | "
                  f"{t['prefill'] * 1e3:8.1f} us {tf['prefill']:6.1f} {100 * tf['prefill'] / 989:5.1f}% | "
                  f"{t['ragged'] / t['prefill']:.1f}x", flush=True)
            del kc, vc, runs
            torch.cuda.empty_cache()


SECTIONS = {"gemm_bench": sec_gemm_bench, "gemm_sweep": sec_gemm_sweep, "misc": sec_misc, "attn": sec_attn,
            "attn_gqa": sec_attn_gqa, "moe": sec_moe, "fp8": sec_fp8, "gemv": sec_gemv, "ragged": sec_ragged,
            "llama": sec_llama, "llama_step": sec_llama_step, "llama_decode": sec_llama_decode,
            "kv_fp8": sec_kv_fp8, "ragged_paged": sec_ragged_paged,
            "paged_prefill": sec_paged_prefill}


def card():
    """The GPU's name and power limit: part of every number this script prints."""
    uuid = f"GPU-{torch.cuda.get_device_properties(0).uuid}"
    r = subprocess.run(["nvidia-smi", "-i", uuid, "--query-gpu=power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return f"{torch.cuda.get_device_name(0)}, power limit {r.stdout.strip() or 'unknown'}"


if __name__ == "__main__":
    names = sys.argv[1:] or list(SECTIONS)
    unknown = [s for s in names if s not in SECTIONS]
    if unknown:
        sys.exit(f"unknown section(s) {unknown}; sections: {' '.join(SECTIONS)}")
    print(f"{card()}, torch {torch.__version__}", flush=True)
    t0 = time.time()
    for s in names:
        SECTIONS[s]()
    print(f"done in {time.time() - t0:.1f}s; FAILS={FAILS}")
    sys.exit(1 if FAILS else 0)
