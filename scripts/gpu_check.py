"""Kernel timings on the GPU: one section per kernel group, each printing `BENCH` lines (CUDA events, median of 20
calls after 5 warm-ups).  The kernels' numerics are checked by the GPU tests under tests/.

usage: python scripts/gpu_check.py [section ...]
  sections: gemm_bench gemm_sweep misc attn moe fp8 gemv ragged (default: all)
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


SECTIONS = {"gemm_bench": sec_gemm_bench, "gemm_sweep": sec_gemm_sweep, "misc": sec_misc, "attn": sec_attn,
            "moe": sec_moe, "fp8": sec_fp8, "gemv": sec_gemv, "ragged": sec_ragged}


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
