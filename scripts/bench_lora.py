"""Multi-LoRA shrink + expand kernels (ops.lora_shrink / ops.lora_expand_) at Llama-3-8B projection shapes.

One call is the delta of one projection for one iteration: shrink, then expand into the projection's output.  The
sweep covers qkv (N 6144, K 4096, three stacked parts), o (4096 x 4096), gate/up (28 672 x 4096, two parts) and down
(4096 x 14 336) at ranks 8, 16 and 64; a decode batch of 128 tokens spread round robin over 1, 8, 32 and 128 adapters,
and one 2048-token prefill with one adapter.

Times are CUDA events around each call with the L2 flushed before it (a 256 MiB write), median of `--reps`.  The bytes
bound is what the call has to move at least: the A and B bytes of the distinct adapters it reads, the x rows read, and
the out rows read and written; GB/s is that over the kernel time, shown also as a share of the H100 SXM data sheet's
3.35 TB/s.  The comparison arm is the eager PyTorch path: per segment, gather the rows, two matmuls, scatter-add.

    python scripts/bench_lora.py --out /tmp/bench_lora.json
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# projection -> (N, K, stacked parts of the rank)
SHAPES = {"qkv": (6144, 4096, 3), "o": (4096, 4096, 1), "gate_up": (28672, 4096, 2), "down": (4096, 14336, 1)}
HBM = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:  # noqa: BLE001
        return f"{torch.cuda.get_device_name()} (power limit not read: {e})"


def segments(T, n_adapters):
    """Round-robin assignment of T rows to n adapters, as the pool lays them out: rows grouped by slot."""
    by = [list(range(a, T, n_adapters)) for a in range(n_adapters)]
    rows = [r for b in by for r in b]
    starts = [0]
    for b in by:
        starts.append(starts[-1] + len(b))
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device="cuda")  # noqa: E731
    return i32(rows), i32(starts), i32(list(range(n_adapters)))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=20)
    p.add_argument("--out", default=None)
    args = p.parse_args()
    from alpa_b200 import ops
    assert torch.cuda.is_available() and ops.native_available(), "bench_lora needs an H100 and the built extension"
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def timed(fn):
        ts = []
        for i in range(args.reps + 3):
            flush.fill_(i & 0xFF)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            if i >= 3:
                ts.append(e0.elapsed_time(e1) * 1e-3)
        return sorted(ts)[len(ts) // 2]

    results = []
    for proj, (N, K, parts) in SHAPES.items():
        for r in (8, 16, 64):
            R = parts * r
            for kind, T, n_ad in [("decode", 128, n) for n in (1, 8, 32, 128)] + [("prefill", 2048, 1)]:
                g = torch.Generator(device="cuda").manual_seed(0)
                x = torch.randn(T, K, device="cuda", generator=g).bfloat16()
                A = (torch.randn(n_ad, R, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
                B = (torch.randn(n_ad, N, R, device="cuda", generator=g) * 0.01).bfloat16()
                scale = torch.ones(n_ad, device="cuda")
                out = torch.randn(T, N, device="cuda", generator=g).bfloat16()
                rows, seg_start, seg_slot = segments(T, n_ad)

                def kernel():
                    ops.fast.lora_expand_(out, ops.fast.lora_shrink(x, A, rows, seg_start, seg_slot), B, scale, rows,
                                          seg_start, seg_slot)
                st = seg_start.tolist()
                segs = [(s, rows[st[s]:st[s + 1]].long()) for s in range(n_ad)]

                def eager():
                    for s, rr in segs:
                        out.index_add_(0, rr, (x[rr] @ A[s].T) @ B[s].T * scale[s].to(out.dtype))
                t_k, t_e = timed(kernel), timed(eager)
                nbytes = n_ad * (R * K + N * R) * 2 + T * K * 2 + 2 * T * N * 2
                results.append({"proj": proj, "N": N, "K": K, "R": R, "r": r, "batch": kind, "tokens": T,
                                "adapters": n_ad, "kernel_us": t_k * 1e6, "eager_us": t_e * 1e6,
                                "bytes": nbytes, "kernel_GBps": nbytes / t_k / 1e9,
                                "share_of_3.35TBps": nbytes / t_k / HBM, "speedup_vs_eager": t_e / t_k})
                row = results[-1]
                print(f"{proj:8s} r={r:3d} R={R:3d} {kind:7s} T={T:5d} adapters={n_ad:4d}  kernel {t_k * 1e6:8.1f} us "
                      f"{row['kernel_GBps']:7.0f} GB/s ({100 * row['share_of_3.35TBps']:5.1f} %)  eager "
                      f"{t_e * 1e6:8.1f} us  x{row['speedup_vs_eager']:.1f}", flush=True)
    meta = {"card": card(), "reps": args.reps, "timing": "CUDA events, L2 flushed, median"}
    print(json.dumps(meta))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"meta": meta, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
