"""First hardware check of the block-scaled MXFP8 path (gemm_sm90.cu): the on-the-fly quantiser against the
PyTorch reference (bit exact), the block-scaled MXFP8 `wgmma` GEMM against an fp32 matmul of the dequantised
operands, and device-timed throughput next to the per-token x per-channel fp8 GEMM.  Written after the round's GPU
budget was spent: run it in a throw-away process with a timeout (tests/test_zzz_gpu_first_hardware_runs.py does).
    python scripts/gpu_check_mxfp8.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from alpa_b200 import ops
    from alpa_b200.ops import primitives as P
    dry = not torch.cuda.is_available()                   # CPU dry run of this script's own logic: reference as "kernel"
    dev = "cpu" if dry else "cuda"
    if dry:
        class C:                                          # noqa: N801
            quantize_mxfp8 = staticmethod(P._quantize_mxfp8_ref)

            @staticmethod
            def gemm_mxfp8_q(q, sf, wq, wsf, b, act):
                y = P.dequantize_mxfp8(q, sf) @ P.dequantize_mxfp8(wq, wsf).t() + (0 if b is None else b.float())
                return (torch.relu(y) if act == 2 else y).to(torch.bfloat16)
    else:
        C = ops.native_module()
    torch.manual_seed(0)
    fails = []
    for (M, N, K) in ((128, 128, 128), (256, 384, 512), (200, 264, 160), (1024, 2560, 2560), (77, 8, 96)):
        x = (torch.randn(M, K, device=dev) * torch.logspace(-2, 2, K, device=dev)[None]).to(torch.bfloat16)
        w = (torch.randn(N, K, device=dev) * 0.05).to(torch.bfloat16)
        b = torch.randn(N, device=dev).to(torch.bfloat16)
        # quantiser: bit exact against the reference
        q, sf = C.quantize_mxfp8(x)
        q_ref, sf_ref = P._quantize_mxfp8_ref(x)
        if not torch.equal(q.view(torch.uint8), q_ref.view(torch.uint8)) or not torch.equal(sf, sf_ref):
            fails.append(f"quantize M{M} K{K}: q mismatches {(q.view(torch.uint8) != q_ref.view(torch.uint8)).sum().item()} "
                         f"sf mismatches {(sf != sf_ref).sum().item()}")
        wq, wsf = C.quantize_mxfp8(w)
        for act in ("none", "relu"):
            y = C.gemm_mxfp8_q(q, sf, wq, wsf, b, P._ACT_IDS[act]).float()
            ref = P.dequantize_mxfp8(q_ref, sf_ref) @ P.dequantize_mxfp8(*P._quantize_mxfp8_ref(w)).t() + b.float()
            ref = torch.relu(ref) if act == "relu" else ref
            err = (y - ref).abs().max().item()
            tol = 0.01 * ref.abs().max().item() + 0.02                       # bf16 output rounding
            print(f"mxfp8 gemm M{M} N{N} K{K} {act}: max err {err:.4f} (tol {tol:.4f})", flush=True)
            if not err <= tol:
                fails.append(f"gemm M{M} N{N} K{K} {act}: err {err} > {tol}")
    if dry:
        print("mxfp8 check (cpu dry run):", "FAILED " + "; ".join(fails) if fails else "ok", flush=True)
        return 1 if fails else 0
    # throughput (device timed)
    M = N = K = 8192
    x = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
    w = torch.randn(N, K, device=dev, dtype=torch.bfloat16)
    q, sf = C.quantize_mxfp8(x)
    wq, wsf = C.quantize_mxfp8(w)

    def timeit(fn, iters=10):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(iters):
            fn()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) / iters
    t = timeit(lambda: C.gemm_mxfp8_q(q, sf, wq, wsf, None, 0))
    print(f"mxfp8 gemm 8192^3: {t:.3f} ms = {2 * M * N * K / t / 1e9:.0f} TFLOPS (operands pre-quantised)", flush=True)
    print("mxfp8 check:", "FAILED " + "; ".join(fails) if fails else "ok", flush=True)
    return 1 if fails else 0


if __name__ == "__main__":
    sys.exit(main())
