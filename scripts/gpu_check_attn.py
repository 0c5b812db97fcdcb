"""Attention kernel checks (numerics vs fp32 PyTorch reference + speed)."""
import math

import torch

from alpa_b200 import ops
_C = ops.native_module()

dev = "cuda"


def ref_attn(q, k, v, scale, causal):
    qf, kf, vf = (t.float().permute(0, 2, 1, 3) for t in (q, k, v))  # [B,h,S,D]
    s = torch.matmul(qf, kf.transpose(-1, -2)) * scale
    if causal:
        Sq, Sk = s.shape[-2:]
        mask = torch.ones(Sq, Sk, device=s.device, dtype=torch.bool).tril(Sk - Sq)
        s = s.masked_fill(~mask, float("-inf"))
    lse = torch.logsumexp(s, dim=-1)
    p = torch.softmax(s, dim=-1)
    o = torch.matmul(p, vf).permute(0, 2, 1, 3)
    return o, lse


def run(check, timeit, FAILS, bwd=True):
    torch.manual_seed(1)
    cases = [(2, 4, 128, 128, 64, False), (2, 4, 256, 256, 64, False), (1, 3, 384, 384, 64, True),
             (2, 2, 200, 200, 64, False), (1, 2, 328, 328, 64, True), (2, 2, 256, 256, 128, False),
             (1, 2, 512, 512, 128, True), (1, 2, 256, 256, 80, False), (1, 4, 1024, 1024, 64, False),
             (1, 2, 128, 512, 64, False), (2, 2, 100, 300, 64, True), (1, 2, 64, 200, 128, True)]
    for (B, H, Sq, Sk, D, causal) in cases:
        qkv = torch.randn(B, max(Sq, Sk), 3, H, D, device=dev, dtype=torch.bfloat16)
        q, k, v = qkv[:, :Sq, 0], qkv[:, :Sk, 1], qkv[:, :Sk, 2]
        scale = 1.0 / math.sqrt(D)
        tag = f"B{B} H{H} Sq{Sq} Sk{Sk} D{D} causal={int(causal)}"
        try:
            o, lse = _C.attention_fwd(q, k, v, scale, causal)
            torch.cuda.synchronize()
        except Exception as ex:  # noqa
            print(f"FAIL attn fwd {tag}: {ex}")
            FAILS.append("attn-exc")
            return
        o_ref, lse_ref = ref_attn(q, k, v, scale, causal)
        check(f"attn fwd o {tag}", o, o_ref, 2e-2, 2e-2)
        check(f"attn fwd lse {tag}", lse, lse_ref, 2e-2, 1e-3)
        if bwd and hasattr(_C, "attention_bwd"):
            do = torch.randn_like(o)
            qf, kf, vf = (t.float().detach().requires_grad_(True) for t in (q, k, v))
            o2, _ = ref_attn(qf, kf, vf, scale, causal)
            o2.backward(do.float())
            try:
                dq, dk, dv = _C.attention_bwd(do, q, k, v, o, lse, scale, causal)
                torch.cuda.synchronize()
            except Exception as ex:  # noqa
                print(f"FAIL attn bwd {tag}: {ex}")
                FAILS.append("attn-bwd-exc")
                return
            check(f"attn bwd dq {tag}", dq, qf.grad, 5e-2, 3e-2)
            check(f"attn bwd dk {tag}", dk, kf.grad, 5e-2, 3e-2)
            check(f"attn bwd dv {tag}", dv, vf.grad, 5e-2, 3e-2)
    # device-side KV length (prefill into a cache): only the first kv_len keys are visible, the causal shift uses kv_len
    for (B, H, Sq, Smax, kvl, D, causal) in [(2, 2, 40, 256, 170, 64, True), (1, 3, 64, 192, 100, 128, False)]:
        q = torch.randn(B, Sq, H, D, device=dev, dtype=torch.bfloat16)
        k = torch.randn(B, Smax, H, D, device=dev, dtype=torch.bfloat16)
        v = torch.randn(B, Smax, H, D, device=dev, dtype=torch.bfloat16)
        scale = 1.0 / math.sqrt(D)
        o, lse = _C.attention_fwd(q, k, v, scale, causal, torch.tensor([kvl], device=dev, dtype=torch.int32))
        o_ref, lse_ref = ref_attn(q, k[:, :kvl], v[:, :kvl], scale, causal)
        tag = f"kv_len B{B} H{H} Sq{Sq} Smax{Smax} kv_len{kvl} D{D} causal={int(causal)}"
        check(f"attn fwd o {tag}", o, o_ref, 2e-2, 2e-2)
        check(f"attn fwd lse {tag}", lse, lse_ref, 2e-2, 1e-3)
    # the 64-query-tile configuration the self-check falls back to (selected per process by ALPA_B200_ATTN_FWD)
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, ALPA_B200_ATTN_FWD="gen2", PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-m", "alpa_b200.ops.selfcheck", "attention_fwd"], env=env, cwd=root,
                       capture_output=True, text=True, timeout=300)
    line = (r.stdout.strip().splitlines() or ["no output"])[-1]
    print(f"attn fwd 64-query tiles: {line}")
    if r.returncode != 0 or " ok" not in line:
        FAILS.append("attn-gen2")
    # speed (GPT-1.3B: 32 heads x 64; 15B: 40 heads x 128)
    flush = torch.empty(256 * 1024 * 1024, device=dev, dtype=torch.uint8)
    for (B, H, S, D, causal) in [(8, 32, 1024, 64, False), (8, 32, 1024, 64, True), (8, 40, 1024, 128, False),
                                 (2, 32, 4096, 64, False)]:
        qkv = torch.randn(B, S, 3, H, D, device=dev, dtype=torch.bfloat16)
        q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
        scale = 1.0 / math.sqrt(D)
        t = timeit(lambda: _C.attention_fwd(q, k, v, scale, causal), flush=flush)
        fl = 4 * B * H * S * S * D * (0.5 if causal else 1.0)
        print(f"BENCH attn fwd B{B} H{H} S{S} D{D} causal={int(causal)}: {t:.3f} ms {fl / t / 1e9:.1f} TFLOPS", flush=True)
        try:
            import torch.nn.functional as F
            qq, kk, vv = (x.transpose(1, 2) for x in (q, k, v))
            t2 = timeit(lambda: F.scaled_dot_product_attention(qq, kk, vv, is_causal=causal), flush=flush)
            print(f"BENCH sdpa(lib) fwd same: {t2:.3f} ms {fl / t2 / 1e9:.1f} TFLOPS", flush=True)
        except Exception as ex:  # noqa
            print("sdpa unavailable", ex)
        if bwd and hasattr(_C, "attention_bwd"):
            o, lse = _C.attention_fwd(q, k, v, scale, causal)
            do = torch.randn_like(o)
            t = timeit(lambda: _C.attention_bwd(do, q, k, v, o, lse, scale, causal), flush=flush)
            print(f"BENCH attn bwd B{B} H{H} S{S} D{D} causal={int(causal)}: {t:.3f} ms {2.5 * fl / t / 1e9:.1f} TFLOPS", flush=True)
