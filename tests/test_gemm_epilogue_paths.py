"""The bf16 GEMM's two epilogue paths (gemm_sm90.cu): the fast kinds, which stage the tile in shared memory and write
it with TMA stores, and the generic register-store epilogue that every other output takes.

The GPU tests run each fast kind (plain store, bias, bias + GELU + aux_out, dGELU from aux_in) and the generic path on
the same inputs (`epilogue="generic"` forces the latter) and require bitwise-equal outputs: the arithmetic is the same,
only where values are staged differs.  Outputs and aux_out sit inside NaN sentinels that must stay bitwise unchanged,
the shapes have M and N tails on both tile widths (including a last tile with a single 8-column strip), a batch with a
padded batch stride, and more tiles than SMs, so a CTA stores one tile while it loads the next.  Outputs a TMA map cannot
describe (a row stride that is not a multiple of 8 elements, a base that is not 16-byte aligned) must take the generic
path and give the same result.

The CPU test compiles gemm_sm90.cu with the build's flags and bounds the machine code of each fast instantiation: the
generic epilogue, fully unrolled with every runtime option, is 130 KB (128-wide tiles) and 248 KB (256-wide tiles).
"""
import os
import subprocess
import sys

import pytest
import torch

from alpa_b200.ops import build

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gemm_numerics import Sentinel, aux_in_values, padded  # noqa: E402

BF16 = torch.bfloat16
ACT_GELU, ACT_DGELU = 1, 3

# (M, N, K, batch, block_n): tails on both widths; 153 and 136 tiles (> 132 SMs); batch 3 with padded batch stride
SHAPES = [
    (2104, 2056, 264, 1, 256),   # 17 x 9 tiles; the last N-block holds 8 columns, so 3 of its 4 chunks are skipped
    (2104, 1000, 192, 1, 128),   # 17 x 8 tiles; the last N-block holds 104 columns (a full and a partial chunk)
    (1100, 520, 128, 3, 0),      # batch 3, 9 M-blocks, N tail
    (64, 136, 72, 1, 256),       # one tile, M smaller than a warpgroup's 64 rows
]
# (kind, trans_a, trans_b): the operand majors the training step runs each kind with (forward, dgrad, wgrad)
KINDS = [("store", ta, tb) for ta in (False, True) for tb in (False, True)] + [
    ("bias", False, False), ("bias_gelu_aux", False, False), ("dgelu", False, True)]


def _operands(M, N, K, batch, ta, tb, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lead = (batch,) if batch > 1 else ()
    a = torch.randn(*lead, *((K, M) if ta else (M, K)), device="cuda", generator=g).to(BF16)
    b = (torch.randn(*lead, *((K, N) if tb else (N, K)), device="cuda", generator=g) * K ** -0.5).to(BF16)
    return padded(a), padded(b), g


def _run(C, kind, a, b, ta, tb, shape, block_n, g, epilogue, make=None):
    """One GEMM of `kind`; returns the wrapped outputs (out, aux_out or None).  `make(shape)` wraps a NaN buffer around
    each output-shaped tensor (a Sentinel by default); aux_in and aux_out share the output's layout."""
    M, N = shape[-2:]
    batch = shape[0] if len(shape) == 3 else None
    make = make or (lambda s: Sentinel(s, BF16))
    out = make(shape)
    kw = {}
    aux = None
    if kind in ("bias", "bias_gelu_aux"):
        kw["bias"] = torch.randn(N, device="cuda", generator=g).to(BF16)
    if kind == "bias_gelu_aux":
        aux = make(shape)
        kw.update(aux_out=aux.view, act=ACT_GELU)
    if kind == "dgelu":
        zin = make(shape)
        zin.view.copy_(aux_in_values(M, N, g, "cuda", batch))
        kw.update(aux_in=zin.view, act=ACT_DGELU)
    C.gemm(a, b, ta, tb, out=out.view, block_n=block_n, epilogue=epilogue, **kw)
    return out, aux


def _bits(t):
    return t.contiguous().view(torch.int16)


def _native():
    from alpa_b200 import ops
    return ops.native_module()


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,batch,block_n", SHAPES)
@pytest.mark.parametrize("kind,ta,tb", KINDS, ids=[f"{k}-A{'mn' if ta else 'k'}-B{'mn' if tb else 'k'}"
                                                   for k, ta, tb in KINDS])
def test_fast_epilogue_matches_generic_bitwise(kind, ta, tb, M, N, K, batch, block_n):
    C = _native()
    shape = (batch, M, N) if batch > 1 else (M, N)
    seed = M + N + K + batch + block_n
    results = {}
    for epilogue in ("auto", "generic"):
        a, b, g = _operands(M, N, K, batch, ta, tb, seed)
        results[epilogue] = _run(C, kind, a, b, ta, tb, shape, block_n, g, epilogue)
    torch.cuda.synchronize()
    (out_f, aux_f), (out_g, aux_g) = results["auto"], results["generic"]
    what = f"{kind} {shape} K{K} block_n={block_n} ta={ta} tb={tb}"
    assert out_f.untouched_outside(), f"{what}: fast epilogue wrote outside the output"
    assert out_g.untouched_outside(), f"{what}: generic epilogue wrote outside the output"
    assert not torch.isnan(out_f.view.float()).any(), f"{what}: output elements never written"
    assert torch.equal(_bits(out_f.view), _bits(out_g.view)), f"{what}: fast and generic outputs differ"
    if aux_f is not None:
        assert aux_f.untouched_outside(), f"{what}: fast epilogue wrote outside aux_out"
        assert torch.equal(_bits(aux_f.view), _bits(aux_g.view)), f"{what}: fast and generic aux_out differ"


class _Strided:
    """An [M, N] bf16 output view in a NaN buffer whose row stride is ld and whose first element is `col0` elements
    into the row (col0 = 2 gives a 4-byte but not 16-byte aligned base)."""

    def __init__(self, shape, ld, col0):
        M, N = shape
        self.buf = torch.full((M + 1, ld), float("nan"), device="cuda", dtype=BF16)
        self.view = self.buf[:M, col0:col0 + N]
        self.before = self.buf.clone()

    def untouched_outside(self):
        mask = torch.ones_like(self.buf, dtype=torch.bool)
        mask[:self.view.shape[0], self.view.storage_offset():self.view.storage_offset() + self.view.shape[1]] = False
        return torch.equal(self.buf.view(torch.int16)[mask], self.before.view(torch.int16)[mask])


@pytest.mark.gpu
@pytest.mark.parametrize("ld,col0", [(1010, 0), (1016, 2)], ids=["ldc-not-multiple-of-8", "base-not-16B-aligned"])
@pytest.mark.parametrize("kind", ["store", "bias_gelu_aux"])
def test_outputs_without_a_tma_map_take_the_generic_path(kind, ld, col0):
    C = _native()
    M, N, K = 2104, 1000, 192
    a, b, g = _operands(M, N, K, 1, False, False, seed=7)
    ref, ref_aux = _run(C, kind, a, b, False, False, (M, N), 256, g, "auto")
    a, b, g = _operands(M, N, K, 1, False, False, seed=7)
    out, aux = _run(C, kind, a, b, False, False, (M, N), 256, g, "auto", make=lambda s: _Strided(s, ld, col0))
    torch.cuda.synchronize()
    what = f"{kind} ld={ld} col0={col0}"
    assert out.untouched_outside(), f"{what}: write outside the output"
    assert torch.equal(_bits(out.view), _bits(ref.view)), f"{what}: output differs from the fast path's"
    if aux is not None:
        assert aux.untouched_outside(), f"{what}: write outside aux_out"
        assert torch.equal(_bits(aux.view), _bits(ref_aux.view)), f"{what}: aux_out differs from the fast path's"


def _text_sizes(obj):
    """{kernel symbol: .text size in bytes} from `cuobjdump -elf`."""
    cuobjdump = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    r = subprocess.run([cuobjdump, "-elf", str(obj)], capture_output=True, text=True, check=True)
    sizes = {}
    for line in r.stdout.splitlines():
        f = line.split()
        if len(f) > 3 and f[-1].startswith(".text._ZN2ab16gemm_sm90_kernel"):
            sym = f[-1][len(".text."):]
            sizes[sym] = max(sizes.get(sym, 0), int(f[2], 16))
    return sizes


# Largest .text allowed per fast kind (EPI template argument) and tile width, measured with CUDA 12.9 plus headroom:
# store 13 / 17 KB, bias 16 / 23 KB, bias + GELU + aux_out 45 / 80 KB, dGELU 50 / 91 KB (128- / 256-wide tiles).
# GELU and its derivative are straight-line erff / expf code for each of the thread's 64 or 128 values.
TEXT_BOUND = {(1, 128): 24 << 10, (1, 256): 32 << 10, (2, 128): 24 << 10, (2, 256): 32 << 10,
              (3, 128): 64 << 10, (3, 256): 112 << 10, (4, 128): 64 << 10, (4, 256): 112 << 10}


@pytest.mark.skipif(not os.path.exists(build.NVCC), reason="nvcc not available")
def test_fast_epilogue_code_size(tmp_path):
    obj = tmp_path / "gemm.o"
    cmd = [build.NVCC, *build.NVCC_FLAGS, f"-I{build.KERNEL_SRC}", "-c", str(build.KERNEL_SRC / "gemm_sm90.cu"),
           "-o", str(obj)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sizes = _text_sizes(obj)
    # gemm_sm90_kernel<BLOCK_N, MODE, A_MAJOR, B_MAJOR, EPI>: _ZN2ab16gemm_sm90_kernelILi<BN>ELi<MODE>ELj<A>ELj<B>ELi<EPI>E
    fast = {}
    for sym, size in sizes.items():
        args = sym[len("_ZN2ab16gemm_sm90_kernelI"):].split("E")[:5]
        bn, mode, _, _, epi = (int(x.lstrip("LijL")) for x in args)
        if mode == 0 and epi != 0:
            fast[sym] = (bn, epi, size)
    # store on all four majors, bias and bias + GELU + aux_out (forward), dGELU (dgrad), on both tile widths
    assert len(fast) == 2 * (4 + 1 + 1 + 1), sorted(fast)
    over = {s: (sz, TEXT_BOUND[(epi, bn)]) for s, (bn, epi, sz) in fast.items() if sz > TEXT_BOUND[(epi, bn)]}
    assert not over, over
