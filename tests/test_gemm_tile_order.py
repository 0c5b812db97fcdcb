"""Tile order of the persistent bf16 GEMM (gemm_sm90.cu `tile_coords`) and the wgmma pipeline of its kernels.

The GPU tests run shapes that take the edge paths of the banded tile order: more tiles than SMs, an M-block count that
is not a multiple of the band height, M and N tails on both tile widths, a batch, and a rotated M-block order.  The
output starts as NaN, so a tile that is never written fails, and each shape also runs with `accumulate=True` on a known
base, so a tile written twice fails.

The CPU test compiles the wgmma translation units with the build's flags and checks that ptxas did not serialize
wgmma (warning C7510, caused by any function call such as printf inside a kernel).
"""
import os
import subprocess

import pytest
import torch

from alpa_b200.ops import build

# (M, N, K, batch, trans_a, trans_b, block_n)
SHAPES = [
    (2104, 2048, 256, 1, False, False, 256),   # 17 M-blocks (bands of 16 and 1, M tail) x 8 N-blocks: 136 tiles > 132 SMs
    (2104, 2048, 256, 1, True, True, 256),     # same order with both operands MN-major
    (2104, 1000, 192, 1, False, True, 256),    # N tail on 256-wide tiles
    (2104, 1000, 192, 1, True, False, 128),    # N tail on 128-wide tiles, 17 x 8 tiles
    (4224, 520, 128, 1, False, False, 128),    # 33 M-blocks: two full bands and a band of one
    (1100, 520, 128, 3, False, False, 0),      # batch 3, 9 M-blocks (a partial band in every batch)
]


def _operands(M, N, K, batch, ta, tb, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lead = (batch,) if batch > 1 else ()
    a = torch.randn(*lead, *((K, M) if ta else (M, K)), device="cuda", dtype=torch.bfloat16, generator=g)
    b = torch.randn(*lead, *((K, N) if tb else (N, K)), device="cuda", dtype=torch.bfloat16, generator=g)
    A = a.float().transpose(-1, -2) if ta else a.float()
    B = b.float() if tb else b.float().transpose(-1, -2)
    return a, b, A @ B


def _assert_close(got, ref, K, what):
    got = got.float()
    assert torch.isfinite(got).all(), f"{what}: {(~torch.isfinite(got)).sum().item()} elements never written"
    err = (got - ref).abs()
    bad = (err > 0.05 * K ** 0.5 + 2e-2 * ref.abs()).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} elements off, max abs err {err.max().item():.4g}"


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,batch,ta,tb,block_n", SHAPES)
def test_every_tile_written_once(M, N, K, batch, ta, tb, block_n):
    from alpa_b200 import ops
    C = ops.native_module()
    a, b, ref = _operands(M, N, K, batch, ta, tb, seed=M + N + K + batch)
    shape = (batch, M, N) if batch > 1 else (M, N)

    out = torch.full(shape, float("nan"), device="cuda", dtype=torch.bfloat16)
    C.gemm(a, b, ta, tb, out=out, block_n=block_n)
    torch.cuda.synchronize()
    _assert_close(out, ref, K, f"gemm {shape} K{K} ta={ta} tb={tb} block_n={block_n}")

    base = torch.randn(shape, device="cuda", dtype=torch.float32)
    acc = base.clone()
    C.gemm(a, b, ta, tb, out=acc, accumulate=True, block_n=block_n)
    torch.cuda.synchronize()
    _assert_close(acc - base, ref, K, f"gemm accumulate {shape} K{K} ta={ta} tb={tb} block_n={block_n}")


@pytest.mark.gpu
@pytest.mark.parametrize("rotate", [0, 5, 16])
def test_rotated_m_blocks(rotate):
    """gemm_wait_a applies `m_block_rotate`; with every M-block owned locally it never waits on a flag."""
    from alpa_b200 import ops
    C = ops.native_module()
    M, N, K = 2104, 2048, 256
    a, w, ref = _operands(M, N, K, 1, False, False, seed=rotate)
    flags = torch.zeros(64, device="cuda", dtype=torch.int32)
    m_blocks = -(-M // 128)
    # gemm_wait_a allocates its output: leave NaN in the block the caching allocator hands back next
    torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
    out = C.gemm_wait_a(a, w, False, flags.data_ptr(), 1, 0, m_blocks, rotate, None, None, 0)
    torch.cuda.synchronize()
    _assert_close(out, ref, K, f"gemm_wait_a rotate={rotate}")


@pytest.mark.skipif(not os.path.exists(build.NVCC), reason="nvcc not available")
@pytest.mark.parametrize("unit", ["gemm_sm90.cu", "attention_sm90.cu"])
def test_wgmma_not_serialized(unit, tmp_path):
    cmd = [build.NVCC, *build.NVCC_FLAGS, f"-I{build.KERNEL_SRC}", "-c", str(build.KERNEL_SRC / unit),
           "-o", str(tmp_path / "unit.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "C7510" not in r.stdout + r.stderr, r.stdout + r.stderr
