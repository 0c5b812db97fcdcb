"""The fp8 KV cache (`OPTConfig(kv_cache_dtype="fp8")`, `ops.Fp8KV`) without a GPU: the reference quantiser against
the format's definition, and the serving paths over an fp8 cache through the PyTorch references -- cached decode and
the graph decode step against one-pass recompute, chunked prefill, ragged batches against solo generation, beam-search
reordering, tensor parallelism, a coarse fp8-against-bf16 logit bound, and the unchanged bf16 default.

Every query attends to the cache's values float(q) * s, its own token's included, so these equalities hold up to
rounding.  The prefill attends to those values rounded to bf16 (the scratch its attention kernel reads), the decode
to the fp32 values, which sets the tolerance of the decode comparisons."""
import os
import sys

import numpy as np
import pytest
import torch

from alpa_b200 import ops
from alpa_b200.model.opt_model import DecoderLM, OPTConfig
from alpa_b200.ops import primitives as P
from alpa_b200.serve.generator import Generator
from alpa_b200.testing import assert_allclose

V = 90


def _cfg(arch, kv=None, **kw):
    if arch == "codegen":
        kw.setdefault("rotary_dim", 8)
    return OPTConfig(arch=arch, vocab_size=V, hidden_size=64, num_hidden_layers=2, num_attention_heads=4,
                     num_key_value_heads=kv, ffn_dim=96, dtype=torch.float32, **kw)


def _model(arch, kv=None, cache="fp8", seed=5):
    return DecoderLM(_cfg(arch, kv, kv_cache_dtype=cache), device="cpu", seed=seed)


# ---------------------------------------------------------------------------------------------------------------- format
def _e4m3_values():
    """Every finite non-negative e4m3fn value (exponent bias 7, no infinities, 0x7F is NaN) with its code."""
    vals = []
    for code in range(0x7F):
        e, m = code >> 3, code & 7
        vals.append((m / 8.0 * 2.0 ** -6) if e == 0 else (1 + m / 8.0) * 2.0 ** (e - 7))
    return np.array(vals)


def _oracle(x):
    """(codes, scales) of rows x [N, D] from the definition: s = max(amax, 1e-8) / 448 in fp32, then x / s in fp32
    rounded to the nearest e4m3 value, ties to the even code."""
    table = _e4m3_values()
    xf = x.float().numpy()
    amax = np.maximum(np.abs(xf).max(-1), np.float32(1e-8)).astype(np.float32)
    s = (amax / np.float32(448.0)).astype(np.float32)
    y = (xf / s[:, None]).astype(np.float32).astype(np.float64)
    a = np.abs(y)
    idx = np.searchsorted(table, a)                         # table[idx - 1] < a <= table[idx]
    lo, hi = np.clip(idx - 1, 0, 126), np.clip(idx, 0, 126)
    dlo, dhi = a - table[lo], table[hi] - a
    pick = np.where(dlo < dhi, lo, np.where(dhi < dlo, hi, np.where(lo % 2 == 0, lo, hi)))
    codes = pick.astype(np.uint8) | np.where(y < 0, 0x80, 0).astype(np.uint8)
    codes = np.where(a == 0, np.where(np.signbit(y), 0x80, 0), codes).astype(np.uint8)
    return torch.from_numpy(codes), torch.from_numpy(s)


def test_reference_quantiser_matches_definition():
    g = torch.Generator().manual_seed(0)
    D = 128
    rows = [torch.randn(D, generator=g), torch.zeros(D), torch.randn(D, generator=g) * 1e30,
            torch.randn(D, generator=g) * 1e-30, torch.randn(D, generator=g) * 3e4, torch.full((D,), -2.5),
            torch.randn(D, generator=g).clamp(-0.1, 0.1) * 1e-4]
    x = torch.stack(rows).to(torch.bfloat16)
    q, s = P._kv_quant_ref(x)
    codes, s_want = _oracle(x)
    assert torch.equal(s, s_want)
    assert torch.equal(q.view(torch.uint8), codes)
    # the elements at +-amax land on +-448 (rows whose amax is under the 1e-8 floor quantise towards 0)
    amax = x.float().abs().amax(-1)
    amax_at = x.float().abs() == amax[:, None]
    vals = q.float()
    big = amax >= 1e-8
    assert torch.all(vals[amax_at & big[:, None]] == x.float()[amax_at & big[:, None]].sign() * 448.0)
    assert torch.all(vals[amax == 0] == 0) and torch.all(vals[~big].abs() < 1e-6 * 448)
    assert torch.all(s[~big] == torch.tensor(1e-8) / torch.tensor(448.0))


def test_store_load_reference_layout():
    """kv_cache_store writes row start + t of sequence b and the head-major scale; kv_cache_load reads them back as
    bf16(float(q) * s); the slot-addressed form writes `rows`."""
    g = torch.Generator().manual_seed(1)
    B, S, H, D, T = 2, 10, 3, 16, 4
    qkv = torch.randn(B, T, H, 4, D, generator=g).to(torch.bfloat16)
    k, v = qkv[:, :, :, 2], qkv[:, :, :, 3]
    kc, vc = ops.Fp8KV.zeros((B, S, H, D), "cpu"), ops.Fp8KV.zeros((B, S, H, D), "cpu")
    ops.kv_cache_store(k, v, kc, vc, 3)
    qk, sk = P._kv_quant_ref(k)
    assert torch.equal(kc.data[:, 3:7].view(torch.uint8), qk.view(torch.uint8))
    assert torch.equal(kc.scale[:, :, 3:7], sk.transpose(1, 2))
    assert kc.data[:, :3].view(torch.uint8).eq(0).all() and kc.data[:, 7:].view(torch.uint8).eq(0).all()
    out = ops.kv_cache_load(vc, 7)
    assert out.dtype == torch.bfloat16 and out.shape == (B, 7, H, D)
    qv, sv = P._kv_quant_ref(v)
    assert torch.equal(out[:, 3:7], (qv.float() * sv[..., None]).to(torch.bfloat16))
    k1, v1 = ops.Fp8KV.zeros((S + 1, H, D), "cpu"), ops.Fp8KV.zeros((S + 1, H, D), "cpu")
    slots = torch.tensor([9, 0, 4, 5])
    ops.kv_cache_store(k[:1], v[:1], k1, v1, rows=slots)
    assert torch.equal(k1.data[slots].view(torch.uint8), qk[0].view(torch.uint8))
    assert torch.equal(k1.scale[:, slots], sk[0].t())
    with pytest.raises(ValueError):
        ops.kv_cache_store(k, v, kc, vc, rows=slots)


def test_store_kernel_takes_rotated_k_next_to_strided_v():
    """Codegen rotates K into a fresh tensor while V stays a view of the packed projection: the store kernel takes
    the two with their own strides, so such a call is not a layout the kernel rejects."""
    qkv = torch.randn(2, 5, 4, 3, 64).to(torch.bfloat16)
    k, v = qkv[:, :, :, 1].contiguous(), qkv[:, :, :, 2]
    assert k.stride() != v.stride()
    assert P._kv_store_unsupported(k, v) is None


# ---------------------------------------------------------------------------------------------------------------- model
# the tolerance of decode against prefill: the prefill attends to the dequantised rows rounded to bf16
TOL = 2e-3

DECODE_CASES = [("llama", 1), ("llama", 2), ("llama", 4), ("opt", None), ("codegen", None)]


@pytest.mark.parametrize("arch,kv", DECODE_CASES)
def test_cached_decode_and_decode_step_equal_recompute(arch, kv):
    m = _model(arch, kv, seed=4)
    B, T, N = 2, 6, 5
    ids = torch.randint(0, V, (B, T + N), generator=torch.Generator().manual_seed(5))
    full = m.forward(ids, torch.arange(T + N).repeat(B, 1), m.init_cache(B, T + N), 0, last_only=False)
    cache, cache2 = m.init_cache(B, 32), m.init_cache(B, 32)
    m.forward(ids[:, :T], torch.arange(T).repeat(B, 1), cache, 0)
    m.forward(ids[:, :T], torch.arange(T).repeat(B, 1), cache2, 0)
    for t in range(T, T + N):
        pos = torch.full((B, 1), t)
        step = m.forward(ids[:, t:t + 1], pos, cache, t)
        dec = m.decode_step(ids[:, t:t + 1], pos, cache2, torch.tensor(t + 1, dtype=torch.int32))
        assert_allclose(step[:, 0], full[:, t], 1e-5, 1e-5)
        assert_allclose(dec, step, TOL, TOL)
    # the first layer's K / V rows depend on the tokens alone: both paths store the same bytes
    for a, b in zip(cache[0], cache2[0]):
        assert isinstance(a, ops.Fp8KV)
        assert torch.equal(a.data.view(torch.uint8), b.data.view(torch.uint8)) and torch.equal(a.scale, b.scale)


def test_chunked_prefill_equals_single_pass():
    m = _model("llama", 2, seed=6)
    ids = [list(range(3, 3 + 19))]
    a = Generator(m, 1, 40).generate(ids, max_new_tokens=6)
    b = Generator(m, 1, 40, prefill_chunk=4).generate(ids, max_new_tokens=6)
    assert torch.equal(a.sequences, b.sequences)
    B, T = 1, 19
    x = torch.tensor(ids)
    c1, c2 = m.init_cache(B, 32), m.init_cache(B, 32)
    one = m.forward(x, torch.arange(T)[None], c1, 0)
    for s0 in range(0, T, 4):
        s1 = min(T, s0 + 4)
        chunked = m.forward(x[:, s0:s1], torch.arange(s0, s1)[None], c2, s0)
    assert_allclose(chunked, one, 1e-5, 1e-5)
    for a, b in zip(c1[0], c2[0]):                        # the first layer's rows depend on the tokens alone
        assert torch.equal(a.data.view(torch.uint8), b.data.view(torch.uint8)) and torch.equal(a.scale, b.scale)


@pytest.mark.parametrize("arch,kv", [("llama", 1), ("llama", 2), ("opt", None), ("bloom", None), ("codegen", None)])
def test_unequal_prompts_equal_solo_generation(arch, kv):
    m = _model(arch, kv, seed=7)
    prompts = [[5, 6, 7, 8, 9, 10, 11], [12, 13, 14], [20, 21, 22, 23, 24]]
    out = Generator(m, 4, 40).generate(prompts, max_new_tokens=6)
    assert isinstance(Generator(m, 4, 40).model.init_cache_1d(8)[0][0], ops.Fp8KV)
    for i, p in enumerate(prompts):
        solo = Generator(m, 1, 40).generate([p], max_new_tokens=6).sequences[0]
        assert out.sequences[i, :len(solo)].tolist() == solo.tolist()


def test_reorder_cache_moves_data_and_scales_together():
    m = _model("llama", 2, seed=8)
    B, T = 3, 7
    ids = torch.randint(0, V, (B, T), generator=torch.Generator().manual_seed(9))
    cache = m.init_cache(B, 16)
    m.forward(ids, torch.arange(T).repeat(B, 1), cache, 0)
    beam = torch.tensor([2, 0, 0])
    Generator.reorder_cache(cache, beam)
    rebuilt = m.init_cache(B, 16)
    m.forward(ids[beam], torch.arange(T).repeat(B, 1), rebuilt, 0)
    for (k1, v1), (k2, v2) in zip(cache, rebuilt):
        for a, b in ((k1, k2), (v1, v2)):
            assert torch.equal(a.data.view(torch.uint8), b.data.view(torch.uint8)) and torch.equal(a.scale, b.scale)
    out = Generator(m, 4, 40).generate([[3, 4, 5, 6]], max_new_tokens=5, num_beams=3)
    assert out.sequences[0, :4].tolist() == [3, 4, 5, 6] and out.sequences.shape[1] >= 5


@pytest.mark.parametrize("arch,kv", [("llama", 2), ("opt", None)])
def test_fp8_cache_logits_stay_near_bf16_cache_logits(arch, kv):
    """Coarse quality bound: the fp8 cache changes a 2-layer model's logits by at most 5 % of their range."""
    ids = torch.randint(0, V, (2, 24), generator=torch.Generator().manual_seed(10))
    pos = torch.arange(24).repeat(2, 1)
    out = {}
    for cache in ("bf16", "fp8"):
        m = _model(arch, kv, cache=cache, seed=11)
        out[cache] = m.forward(ids, pos, m.init_cache(2, 24), 0, last_only=False)
    err = (out["fp8"] - out["bf16"]).abs().max()
    assert err <= 0.05 * out["bf16"].abs().max(), float(err)


def test_bf16_default_allocates_todays_tensors():
    for kw in ({}, {"kv_cache_dtype": "bf16"}):
        m = DecoderLM(_cfg("llama", 2, **kw), device="cpu")
        assert m.cfg.kv_cache_dtype == "bf16"
        for k, v in m.init_cache(3, 8):
            assert type(k) is torch.Tensor and k.shape == (3, 8, 2, 16) and k.dtype == torch.float32
            assert type(v) is torch.Tensor and v.shape == k.shape
        for k, v in m.init_cache_1d(5):
            assert type(k) is torch.Tensor and k.shape == (6, 2, 16)
    with pytest.raises(ValueError):
        _cfg("opt", kv_cache_dtype="e5m2")


def test_fp8_cache_bytes():
    m = _model("llama", 2)
    bf16 = ops.kv_cache_nbytes(DecoderLM(_cfg("llama", 2), device="cpu").init_cache(2, 8))
    fp8 = ops.kv_cache_nbytes(m.init_cache(2, 8))
    L, B, S, H, D = 2, 2, 8, 2, 16
    assert bf16 == L * 2 * B * S * H * D * 4                 # this test's model computes in fp32
    assert fp8 == L * 2 * B * S * H * (D + 4)


def _tp_worker(rank, world, port):
    """One rank of the tensor-parallel check: with an fp8 cache, tp = world generates what tp = 1 generates."""
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        for arch, kv in (("llama", 2), ("opt", None)):
            cfg = _cfg(arch, kv, kv_cache_dtype="fp8")
            ref = DecoderLM(cfg, device="cpu", seed=5)
            tp = DecoderLM(cfg, device="cpu", group=dist.group.WORLD, seed=5)
            prompts = [[5, 6, 7, 8, 9], [9, 10, 11, 12, 13]]
            o_ref = Generator(ref, 2, 32).generate(prompts, max_new_tokens=5)
            o_tp = Generator(tp, 2, 32).generate(prompts, max_new_tokens=5)
            assert torch.equal(o_ref.sequences, o_tp.sequences), (arch, o_ref.sequences, o_tp.sequences)
        print(f"rank {rank}: fp8 cache tp ok", flush=True)
    finally:
        dist.destroy_process_group()


def test_tensor_parallel_world2():
    import socket
    import subprocess
    here = os.path.dirname(os.path.abspath(__file__))
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    code = ("import sys; sys.path[:0] = [{!r}, {!r}]; import test_kv_cache_fp8 as t; t._tp_worker({{}}, 2, {})"
            .format(os.path.dirname(here), here, port))
    procs = [subprocess.Popen([sys.executable, "-c", code.format(r)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                              text=True) for r in range(2)]
    try:
        outs = [p.communicate(timeout=240)[0] for p in procs]
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
    for r, (p, out) in enumerate(zip(procs, outs)):
        assert p.returncode == 0 and f"rank {r}: fp8 cache tp ok" in out, out[-3000:]
