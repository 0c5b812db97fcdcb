"""The multi-LoRA shrink / expand kernels (lora_sm90.cu) against float64 references with bf16-scaled error budgets, and
multi-LoRA serving on the H100 against models built from merged weights."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_lora_serving import _adapter, _base_hf, _params, _prompts, _run, tiny  # noqa: E402

from alpa_b200 import ops  # noqa: E402
from alpa_b200.model.opt_model import DecoderLM  # noqa: E402
from alpa_b200.ops import primitives  # noqa: E402
from alpa_b200.serve.batching import InputPoolConfig  # noqa: E402
from alpa_b200.serve.generator import load_lora_np  # noqa: E402

pytestmark = pytest.mark.gpu

U = 2.0 ** -8          # bf16 unit roundoff


def _segments(T, sizes, slots, skip_every=0, seed=0):
    """rows / seg_start / seg_slot of segments of the given sizes over a batch of T rows (shuffled rows; every
    `skip_every`-th row left out of every segment)."""
    g = torch.Generator().manual_seed(seed)
    pool = torch.randperm(T, generator=g)
    if skip_every:
        pool = pool[torch.arange(T) % skip_every != 0]
    assert sum(sizes) <= len(pool)
    rows = pool[:sum(sizes)]
    starts = [0]
    for n in sizes:
        starts.append(starts[-1] + n)
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device="cuda")  # noqa: E731
    return rows.to(torch.int32).cuda(), i32(starts), i32(slots)


def _check(T, K, N, R, sizes, slots, nslots, skip_every=0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(T, K, device="cuda", generator=g).bfloat16()
    A = (torch.randn(nslots, R, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    B = (torch.randn(nslots, N, R, device="cuda", generator=g) / R ** 0.5).bfloat16()
    scale = torch.rand(nslots, device="cuda", generator=g) + 0.5
    out = torch.randn(T, N, device="cuda", generator=g).bfloat16()
    rows, seg_start, seg_slot = _segments(T, sizes, slots, skip_every, seed)
    before = out.clone()
    y = ops.fast.lora_shrink(x, A, rows, seg_start, seg_slot)
    assert y.dtype == torch.float32 and y.shape[1:] == (rows.numel(), R)
    ys = y.sum(0).double()
    ops.fast.lora_expand_(out, y, B, scale, rows, seg_start, seg_slot)
    # float64 references
    st = seg_start.tolist()
    for s, slot in enumerate(seg_slot.tolist()):
        r = rows[st[s]:st[s + 1]].long()
        if r.numel() == 0:
            continue
        xr, a, b = x[r].double(), A[slot].double(), B[slot].double()
        y64 = xr @ a.T
        bound = 2.0 ** -16 * (xr.abs() @ a.abs().T) + 1e-30
        assert ((ys[st[s]:st[s + 1]] - y64).abs() <= bound).all(), (K, R, s)
        ref = before[r].double() + scale[slot].double() * (y64 @ b.T)
        budget = U * ref.abs() + 2 * U * scale[slot].double() * (y64.abs() @ b.abs().T) + 1e-6
        err = (out[r].double() - ref).abs()
        assert (err <= budget).all(), (K, N, R, s, float((err / budget).max()))
    untouched = torch.ones(T, dtype=torch.bool, device="cuda")
    untouched[rows.long()] = False
    assert torch.equal(out[untouched], before[untouched])            # bitwise: never read or written
    # the same bits again
    out2 = before.clone()
    y2 = ops.fast.lora_shrink(x, A, rows, seg_start, seg_slot)
    ops.fast.lora_expand_(out2, y2, B, scale, rows, seg_start, seg_slot)
    assert torch.equal(y2, y) and torch.equal(out2, out)


@pytest.mark.parametrize("K", [2048, 4096, 14336])
@pytest.mark.parametrize("R", [8, 48, 64, 192])
def test_decode_segments(K, R):
    # 128 decode rows over 32 adapters (1 to 7 rows each, some empty), many slots
    sizes = [(i * 5) % 8 for i in range(32)]
    _check(160, K, 1024, R, sizes, list(range(0, 64, 2)), 64, skip_every=5, seed=K + R)


@pytest.mark.parametrize("K,N", [(4096, 6144), (14336, 4096), (2048, 1000 // 8 * 8)])
@pytest.mark.parametrize("R", [16, 120, 192])
def test_prefill_segment(K, N, R):
    _check(2048, K, N, R, [2048], [1], 3, seed=K + R)


def test_mixed_prefill_and_decode_segments():
    # one long segment, a few short ones, empty segments, rows of the base model in between
    _check(800, 4096, 4096, 48, [0, 513, 1, 0, 37, 2, 64], [0, 1, 2, 3, 4, 5, 7], 8, skip_every=7)


def test_unsupported_layout_records_one_fallback():
    primitives._FALLBACK_SEEN.clear()
    x = torch.randn(16, 64, device="cuda").bfloat16()
    A = torch.randn(2, 12, 64, device="cuda").bfloat16()             # R = 12: not a multiple of 8
    rows, seg_start, seg_slot = _segments(16, [4], [1])
    for _ in range(2):
        y = ops.fast.lora_shrink(x, A, rows, seg_start, seg_slot)
    want = x[rows.long()].float() @ A[1].float().T
    torch.testing.assert_close(y[0], want, atol=1e-3, rtol=1e-3)
    assert [f[0] for f in primitives.library_fallbacks()] == ["lora_shrink"]
    primitives._FALLBACK_SEEN.clear()


# ------------------------------------------------------------------ serving on the H100
def _serving_cfg(arch, weight_dtype="bf16", dtype=torch.bfloat16):
    return tiny(arch, vocab_size=512, hidden_size=256, num_attention_heads=4, ffn_dim=512, dtype=dtype,
                weight_dtype=weight_dtype)


def _pool():
    return InputPoolConfig(batch_size=256, cache_size=2048, max_cache_per_seq=128, kv_block_size=16)


def _max_err(got, want, keys):
    return max(float((got[k].float().cpu() - want[k].float().cpu()).abs().max()) for k in keys)


@pytest.mark.parametrize("arch,weight_dtype", [("llama", "bf16"), ("llama", "fp8"), ("opt", "bf16")])
def test_serving_matches_merged_weights_on_h100(tmp_path, arch, weight_dtype):
    """Adapters served on the H100 against fp32 models of merged weights on the CPU (the exact oracle): no further
    from it than the served model's base requests are from the fp32 base model, or than bf16 merged weights on the
    H100 are from the oracle.  Base requests of the mixed batch are bitwise those of a batch without adapters."""
    cfg, cfg32 = _serving_cfg(arch, weight_dtype), _serving_cfg(arch, dtype=torch.float32)
    base = _base_hf(cfg32, 1)
    m = DecoderLM(cfg, device="cuda", params=_params(cfg, base))
    deltas = {}
    for k, (name, r) in enumerate((("a", 8), ("b", 16))):
        deltas[name] = _adapter(cfg, str(tmp_path / name), r, 16.0, 20 + k)
        m.load_lora(name, *load_lora_np(cfg, str(tmp_path / name)))
    prompts = _prompts(8, 3, 20, 90, V=512)
    loras = [None, "a", "b", "a", None, "b", "a", "b"]
    none = [None] * len(prompts)
    primitives._FALLBACK_SEEN.clear()
    got, _ = _run(m, prompts, loras, _pool())
    assert not [f for f in primitives.library_fallbacks() if f[0].startswith("lora")]
    plain, _ = _run(m, prompts, none, _pool())
    base_keys = [k for k in got if loras[k[0]] is None]
    for k in base_keys:
        assert torch.equal(got[k], plain[k]), k
    ref, _ = _run(DecoderLM(cfg32, device="cpu", params=_params(cfg32, base)), prompts, none, _pool())
    floor = _max_err(plain, ref, list(plain))
    for name, d in deltas.items():
        keys = [k for k in got if loras[k[0]] == name]
        ref, _ = _run(DecoderLM(cfg32, device="cpu", params=_params(cfg32, base, d)), prompts, none, _pool())
        bf16, _ = _run(DecoderLM(_serving_cfg(arch), device="cuda", params=_params(cfg, base, d)), prompts, none,
                       _pool())
        bound = 2 * max(floor, _max_err(bf16, ref, keys))
        err = _max_err(got, ref, keys)
        print(f"{arch} {weight_dtype} adapter {name}: max |logit error| {err:.4f}, bound {bound:.4f}")
        assert err <= bound, (name, err, bound)
