"""First hardware run of the resharding pack / unpack kernel (pack_sm90.cu) against the PyTorch reference, plus the
device-timed cost of one packed launch next to one `.contiguous()` copy per tile.
    python scripts/gpu_check_pack.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from alpa_b200 import ops
    from alpa_b200.global_env import global_config
    dry = not torch.cuda.is_available()                   # CPU dry run of this script's own logic
    dev = "cpu" if dry else "cuda"
    torch.manual_seed(0)
    fails = []
    x = torch.randn(8, 1024, 2048, device=dev).to(torch.bfloat16)
    f = torch.randn(37, 53, device=dev)
    cases = {
        "column halves (vector path)": [x[b, :, 1024:] for b in range(8)],
        "row + column boxes": [x[1:3, 100:612, 256:512], x[0], x[:, 5:9, :], x[7, 1023, 8:16]],
        "odd sizes (byte path)": [f[:, 3:20], f[5], f[1:30, 52:53]],
        "40 tiles (two launches)": [x[i % 8, i:i + 8, 64:128] for i in range(40)],
    }
    for name, views in cases.items():
        flat = ops.pack_tiles(views)
        global_config.use_native_kernels = False
        ref = ops.pack_tiles(views)                         # PyTorch reference of the same layout
        global_config.use_native_kernels = True
        same = all(torch.equal(flat[o:o + n], ref[o:o + n]) for o, n in _extents(views))   # padding bytes are undefined
        dst = [torch.zeros_like(v) for v in views]
        ops.unpack_tiles(flat, dst)
        back = all(torch.equal(a, b) for a, b in zip(views, dst))
        print(f"pack {name}: packed == reference {same}, round trip {back}", flush=True)
        if not (same and back):
            fails.append(name)
    if not dry:
        views = cases["column halves (vector path)"]
        flat = torch.empty(ops.packed_nbytes(views), dtype=torch.uint8, device=dev)

        def timeit(fn, iters=50):
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                fn()
            e.record()
            torch.cuda.synchronize()
            return s.elapsed_time(e) / iters * 1e3
        t_pack = timeit(lambda: ops.pack_tiles(views, flat))
        t_copy = timeit(lambda: [v.contiguous() for v in views])
        gb = 2 * flat.numel() / 1e9
        print(f"pack 8 x [1024, 1024] bf16 column halves: one launch {t_pack:.1f} us ({gb / t_pack * 1e6:.0f} GB/s) vs "
              f"8 copy launches {t_copy:.1f} us", flush=True)
    tag = "pack check (cpu dry run):" if dry else "pack check:"
    print(tag, "FAILED " + "; ".join(fails) if fails else "ok", flush=True)
    return 1 if fails else 0


def _extents(views):
    off = 0
    for v in views:
        n = v.numel() * v.element_size()
        yield off, n
        off += (n + 15) // 16 * 16


if __name__ == "__main__":
    sys.exit(main())
