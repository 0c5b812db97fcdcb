"""The serving attention kernels against float64 references: `decode_attention` (one new token per sequence, cache
append fused in), `ragged_attention` (a 1-D token batch over a slot-addressed cache) and `attention_cached_` on the
native path.

Every reference is float64 and is computed from the exact bf16 values the kernel read.  Neither kernel rounds P, so
the baseline of `bf16_rule` (tests/test_kernel_numerics.py) is the float64 result rounded to bf16 once.  The prompt
chunk of `attention_cached_` runs the flash-attention forward, whose baseline rounds the unnormalised P as well.

Reads outside what the kernel may read are poisoned: cache rows at or past the valid length, the gaps between ragged
sequences and the scratch row are NaN, and so is the stale cache row the decode kernel overwrites with the new key /
value (it must attend to the appended row from its source).  After a call, the appended row must equal k_new / v_new
bit for bit and every other byte of the cache buffers must be unchanged.

The CPU tests show the rule rejects the wrong results these kernels would produce with a dropped split, a stale
appended row, a 2 % softmax-scale error, a dropped newest key and an ALiBi bias of the wrong sign.
"""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernel_numerics import (BF16, F64, WORST, Checker, _bf, _report, attn_fwd_ref, bf16_rule,  # noqa: E402
                                  visible)

NAN = float("nan")
HARD_LOGIT = 30.0          # the logit of the one key that decides the output in the "hard" inputs


@pytest.fixture(scope="module", autouse=True)
def _print_worst_ratios():
    before = set(WORST)
    yield
    mine = sorted(k for k in WORST if k not in before)
    if mine:
        print("\n[serving attention numerics] worst ratio of kernel error to baseline error:")
        for k in mine:
            print(f"  {k:40s} {WORST[k]:.3f}")


# ---------------------------------------------------------------------------------------------------------------------
# references (float64 on whatever device the inputs live on)
# ---------------------------------------------------------------------------------------------------------------------


def decode_ref(q, k, v, scale):
    """o [B, h, D] float64: softmax(q . k^T * scale) v over all n rows of k / v [B, n, h, D]; q [B, h, D]."""
    s = torch.einsum("bhd,bnhd->bhn", q.to(F64), k.to(F64)) * scale
    return torch.einsum("bhn,bnhd->bhd", torch.softmax(s, -1), v.to(F64))


def ragged_ref(q, k_cache, v_cache, seq_start, ctx_len, scale, alibi=None):
    """o [T, h, D] float64: token t attends to cache rows seq_start[t] + j, j < ctx_len[t], with the bias slope * j;
    tokens with ctx_len 0 give zeros."""
    T, h, D = q.shape
    out = torch.zeros(T, h, D, dtype=F64, device=q.device)
    for t in range(T):
        n, st = int(ctx_len[t]), int(seq_start[t])
        if n <= 0:
            continue
        k = k_cache[st:st + n].to(F64)
        v = v_cache[st:st + n].to(F64)
        s = torch.einsum("hd,nhd->hn", q[t].to(F64), k) * scale
        if alibi is not None:
            s = s + alibi.to(F64)[:, None] * torch.arange(n, dtype=F64, device=q.device)[None, :]
        out[t] = torch.einsum("hn,nhd->hd", torch.softmax(s, -1), v)
    return out


def decode_splits(B, heads, sms):
    """The binding's split count: about two CTAs per SM over the (sequence, head) rows, 1 to 16."""
    return max(1, min(16, (2 * sms + B * heads - 1) // (B * heads)))


def split_ranges(n, splits):
    """The key range [begin, end) of each split for n valid rows (a multiple of 16 keys per split)."""
    per = ((n + splits - 1) // splits + 15) // 16 * 16
    return [(min(i * per, n), min(i * per + per, n)) for i in range(splits)]


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the rule rejects the wrong results of these kernels
# ---------------------------------------------------------------------------------------------------------------------


def _decode_case(B, h, D, n, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, h, D, generator=g).to(BF16)
    k = torch.randn(B, n, h, D, generator=g).to(BF16)
    v = torch.randn(B, n, h, D, generator=g).to(BF16)
    return q, k, v


def test_rule_rejects_decode_attention_defects():
    scale = 128 ** -0.5
    q, k, v = _decode_case(2, 16, 128, 2048, 0)
    ref = decode_ref(q, k, v, scale)
    base = _bf(ref)
    assert not bf16_rule("baseline", base, ref, base)[0]
    splits = decode_splits(2, 16, 132)
    b0, b1 = split_ranges(2048, splits)[-1]
    wrong = {
        "last split dropped": decode_ref(q, k[:, :b0], v[:, :b0], scale),
        "softmax scale off by 2 %": decode_ref(q, k, v, scale * 1.02),
    }
    # kv_len 513 with 16 splits: the last split holds one key
    q2, k2, v2 = _decode_case(1, 32, 80, 513, 1)
    ref2 = decode_ref(q2, k2, v2, 80 ** -0.5)
    assert split_ranges(513, decode_splits(1, 32, 132))[-1] == (512, 513)
    # the stale cache row instead of the appended one
    q3, k3, v3 = _decode_case(3, 4, 80, 77, 2)
    ref3 = decode_ref(q3, k3, v3, 80 ** -0.5)
    g = torch.Generator().manual_seed(3)
    ks, vs = k3.clone(), v3.clone()
    ks[:, -1] = torch.randn(3, 4, 80, generator=g).to(BF16)
    vs[:, -1] = torch.randn(3, 4, 80, generator=g).to(BF16)
    cases = [(ref, base, w, nm) for nm, w in wrong.items()]
    cases.append((ref2, _bf(ref2), decode_ref(q2, k2[:, :512], v2[:, :512], 80 ** -0.5), "one-key last split dropped"))
    cases.append((ref3, _bf(ref3), decode_ref(q3, ks, vs, 80 ** -0.5), "stale appended row"))
    for r, b, w, nm in cases:
        msgs, ratio = bf16_rule(nm, _bf(w), r, b)
        assert msgs, f"{nm}: accepted (ratio {ratio:.2f})"


def test_rule_rejects_ragged_attention_defects():
    g = torch.Generator().manual_seed(4)
    h, D, n = 4, 64, 1000
    kc = torch.randn(n, h, D, generator=g).to(BF16)
    vc = torch.randn(n, h, D, generator=g).to(BF16)
    q = torch.randn(3, h, D, generator=g).to(BF16)
    ss = torch.zeros(3, dtype=torch.int32)
    cl = torch.tensor([n, n - 1, n - 2], dtype=torch.int32)
    alibi = torch.tensor([2.0 ** (-8 * (i + 1) / h) for i in range(h)])
    for ab in (None, alibi):
        ref = ragged_ref(q, kc, vc, ss, cl, D ** -0.5, ab)
        base = _bf(ref)
        assert not bf16_rule("baseline", base, ref, base)[0]
        dropped = ragged_ref(q, kc, vc, ss, cl - 1, D ** -0.5, ab)
        assert bf16_rule("newest key dropped", _bf(dropped), ref, base)[0]
        if ab is not None:
            flipped = ragged_ref(q, kc, vc, ss, cl, D ** -0.5, -ab)
            assert bf16_rule("alibi of the wrong sign", _bf(flipped), ref, base)[0]


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------------


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _hard_scale(q, scale):
    """c such that (c q) . q * scale ~ HARD_LOGIT, per [.., D] row of q."""
    qq = q.float().pow(2).sum(-1, keepdim=True).clamp_min(1e-6)
    return HARD_LOGIT / (scale * qq)


def _decode_inputs(B, h, D, S_max, n, kind, seed):
    """(qkv [B,1,h,3,D], k / v cache buffers [B, S_max + 3, h, D] with rows < n-1 random and the rest NaN)."""
    g = _gen(seed)
    scale = D ** -0.5
    qkv = torch.randn(B, 1, h, 3, D, generator=g, device="cuda").to(BF16)
    kbuf = torch.full((B, S_max + 3, h, D), NAN, device="cuda", dtype=BF16)
    vbuf = torch.full_like(kbuf, NAN)
    kbuf[:, :n - 1] = torch.randn(B, n - 1, h, D, generator=g, device="cuda").to(BF16)
    vbuf[:, :n - 1] = torch.randn(B, n - 1, h, D, generator=g, device="cuda").to(BF16)
    q = qkv[:, 0, :, 0]
    if kind == "hard_new":
        qkv[:, 0, :, 1] = (_hard_scale(q, scale) * q.float()).to(BF16)
    elif kind == "hard_cache0" and n > 1:
        kbuf[:, 0] = (_hard_scale(q, scale) * q.float()).to(BF16)
    return qkv, kbuf, vbuf


def _check_decode_call(ck, key, name, o, q, k_new, v_new, kbuf, vbuf, before_k, before_v, n, scale):
    """o against float64 over rows [0, n) with row n-1 = the new row; the new row written bit for bit; nothing else."""
    kr = before_k[:, :n].clone()
    vr = before_v[:, :n].clone()
    kr[:, n - 1] = k_new.reshape(kr[:, n - 1].shape)
    vr[:, n - 1] = v_new.reshape(vr[:, n - 1].shape)
    ref = decode_ref(q.reshape(q.shape[0], q.shape[-2], q.shape[-1]), kr, vr, scale)
    ck.bf16(key, name, o.reshape(ref.shape), ref, _bf(ref))
    for nm, buf, before, new in (("k", kbuf, before_k, k_new), ("v", vbuf, before_v, v_new)):
        want = before.clone()
        want[:, n - 1] = new.reshape(want[:, n - 1].shape)
        ck.require(torch.equal(buf.view(torch.int16), want.view(torch.int16)),
                   f"{name}: {nm} cache buffer differs from the appended reference outside row {n - 1} or in it")


# (B, heads, D, S_max, kv lengths): B * heads on both sides of 2 x SMs, so the split count covers 16, 1 and values in
# between; lengths of one key, around a half-warp stride (16), around the unrolled stride (64), below 16 x splits (some
# splits empty), long, and S_max (the append goes into the last row).
DECODE_CASES = [
    (1, 8, 128, 2100, [1, 15, 16, 17, 63, 65, 100, 2048, 2100]),
    (2, 4, 8, 256, [1, 16, 63, 100, 256]),
    (2, 16, 80, 600, [1, 17, 65, 130, 513, 600]),
    (4, 16, 64, 2050, [16, 65, 2048]),
    (33, 8, 96, 700, [1, 15, 16, 17, 63, 65, 700]),
    (40, 8, 8, 300, [1, 17, 300]),
    (48, 8, 128, 2048, [2048]),
]
KINDS = ["randn", "hard_new", "hard_cache0"]


@pytest.mark.gpu
@pytest.mark.parametrize("B,h,D,S_max,lens", DECODE_CASES, ids=[f"B{c[0]}-h{c[1]}-D{c[2]}" for c in DECODE_CASES])
def test_decode_attention(B, h, D, S_max, lens):
    from alpa_b200.ops import primitives as P
    ck = Checker()
    scale = D ** -0.5
    splits = decode_splits(B, h, _sms())
    key = f"decode_attention D{D}"
    for n in lens:
        for i, kind in enumerate(KINDS):
            qkv, kbuf, vbuf = _decode_inputs(B, h, D, S_max, n, kind, 1000 * n + 10 * D + i)
            kc, vc = kbuf[:, :S_max], vbuf[:, :S_max]
            bk, bv = kbuf.clone(), vbuf.clone()
            q, kn, vn = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
            kv = torch.tensor([n], dtype=torch.int32, device="cuda")
            o = P.decode_attention(q, kn, vn, kc, vc, kv, scale)
            _check_decode_call(ck, key, f"{key} B{B} h{h} n{n} splits={splits} {kind}", o, q, kn, vn, kbuf, vbuf,
                               bk, bv, n, scale)
    _report(ck)


@pytest.mark.gpu
def test_decode_attention_covers_every_split_regime():
    sms = _sms()
    splits = {decode_splits(c[0], c[1], sms) for c in DECODE_CASES}
    assert 1 in splits and 16 in splits and any(1 < s < 16 for s in splits), splits
    short = [(c, n) for c in DECODE_CASES for n in c[4]
             if any(b == e for b, e in split_ranges(n, decode_splits(c[0], c[1], sms)))]
    assert short, "no case leaves a split without keys"


@pytest.mark.gpu
def test_decode_attention_unequal_new_strides():
    """k_new and v_new with different strides take the primitive's copy path."""
    from alpa_b200.ops import primitives as P
    B, h, D, S_max, n = 2, 8, 64, 300, 129
    ck = Checker()
    qkv, kbuf, vbuf = _decode_inputs(B, h, D, S_max, n, "randn", 7)
    kc, vc = kbuf[:, :S_max], vbuf[:, :S_max]
    bk, bv = kbuf.clone(), vbuf.clone()
    q, kn = qkv[:, :, :, 0], qkv[:, :, :, 1]
    vn = torch.randn(B, 1, h, D, generator=_gen(8), device="cuda").to(BF16)
    assert kn.stride() != vn.stride()
    kv = torch.tensor([n], dtype=torch.int32, device="cuda")
    o = P.decode_attention(q, kn, vn, kc, vc, kv, D ** -0.5)
    _check_decode_call(ck, "decode_attention D64", "decode_attention unequal k_new / v_new strides", o, q, kn, vn,
                       kbuf, vbuf, bk, bv, n, D ** -0.5)
    _report(ck)


@pytest.mark.gpu
@pytest.mark.parametrize("B,h,D", [(1, 8, 128), (33, 8, 64)], ids=["splits16", "splits1"])
def test_decode_attention_graph_replay(B, h, D):
    """One captured call replayed at five consecutive lengths, kv_len incremented on the device: every output against
    float64 (the split arrival counters must be reset by each launch)."""
    from alpa_b200.ops import primitives as P
    ck = Checker()
    S_max, n0 = 512, 200
    scale = D ** -0.5
    splits = decode_splits(B, h, _sms())
    assert (splits > 1) == (B == 1)
    qkv, kbuf, vbuf = _decode_inputs(B, h, D, S_max, n0, "randn", 21 + B)
    kc, vc = kbuf[:, :S_max], vbuf[:, :S_max]
    q, kn, vn = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
    kv = torch.tensor([n0], dtype=torch.int32, device="cuda")
    # warm-up on scratch tensors of the same shape: the binding's arrival counters exist before the capture
    P.decode_attention(q, kn, vn, kc.clone(), vc.clone(), kv.clone(), scale)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        o = P.decode_attention(q, kn, vn, kc, vc, kv, scale)
    g = _gen(22)
    for step in range(5):
        n = n0 + step
        if step:
            kv += 1
            qkv.copy_(torch.randn(qkv.shape, generator=g, device="cuda").to(BF16))
        bk, bv = kbuf.clone(), vbuf.clone()
        graph.replay()
        torch.cuda.synchronize()
        ck.require(int(kv) == n, f"kv_len {int(kv)} != {n}")
        _check_decode_call(ck, f"decode_attention D{D}", f"decode graph replay B{B} h{h} n{n} splits={splits}", o, q,
                           kn, vn, kbuf, vbuf, bk, bv, n, scale)
    _report(ck)


def _ragged_batch(h, D, chunks, seed, hard=False):
    """A 1-D batch over one cache.  `chunks`: (sequence length, query tokens) per sequence; the query tokens are the
    last ones of the sequence (a prompt chunk when several, a decode token when one).  Two padding tokens follow.
    Cache rows outside every sequence (the gaps and the scratch row) are NaN.  hard: each single-token sequence's
    newest key is c * q with a logit of about HARD_LOGIT."""
    g = _gen(seed)
    starts, s = [], 5
    for n, _ in chunks:
        starts.append(s)
        s += n + 3
    slots = s + 1
    kc = torch.full((slots, h, D), NAN, device="cuda", dtype=BF16)
    vc = torch.full_like(kc, NAN)
    seq_start, ctx_len, owner = [], [], []
    for i, (st, (n, k)) in enumerate(zip(starts, chunks)):
        kc[st:st + n] = torch.randn(n, h, D, generator=g, device="cuda").to(BF16)
        vc[st:st + n] = torch.randn(n, h, D, generator=g, device="cuda").to(BF16)
        for j in range(n - k, n):
            seq_start.append(st)
            ctx_len.append(j + 1)
            owner.append(i)
    seq_start += [0, 0]
    ctx_len += [0, 0]
    T = len(seq_start)
    qkv = torch.randn(T, h, 3, D, generator=g, device="cuda").to(BF16)
    q = qkv[:, :, 0]
    if hard:
        for t, i in enumerate(owner):
            n, k = chunks[i]
            if k == 1:
                kc[starts[i] + n - 1] = (_hard_scale(q[t], D ** -0.5) * q[t].float()).to(BF16)
    ss = torch.tensor(seq_start, dtype=torch.int32, device="cuda")
    cl = torch.tensor(ctx_len, dtype=torch.int32, device="cuda")
    return q, kc, vc, ss, cl


RAGGED_DIMS = [16, 24, 64, 80, 128, 136, 256]
# (sequence length, query tokens): contexts 1, 127-129 (a prompt chunk), 128 and 4000 (decode tokens); the long batch
# adds a 16 000-key decode token, whose score buffer (64 KB) takes the > 48 KB dynamic shared memory path
RAGGED_SHORT = [(1, 1), (129, 3), (128, 1), (4000, 1), (40, 40)]
RAGGED_LONG = [(16000, 1), (300, 2), (1, 1)]


def _ragged_smem(D, max_ctx):
    return 4 * (D + 8 + (128 // (D // 2)) * D + max_ctx)


@pytest.mark.gpu
@pytest.mark.parametrize("D", RAGGED_DIMS)
def test_ragged_attention(D):
    from alpa_b200 import ops
    ck = Checker()
    h = 4
    alibi = torch.tensor([2.0 ** (-8 * (i + 1) / h) for i in range(h)], device="cuda")
    smem = []
    for bi, (chunks, hard) in enumerate([(RAGGED_SHORT, False), (RAGGED_SHORT, True), (RAGGED_LONG, False)]):
        q, kc, vc, ss, cl = _ragged_batch(h, D, chunks, 100 * D + bi, hard)
        mc = max(n for n, _ in chunks)
        smem.append(_ragged_smem(D, mc))
        bk, bv = kc.clone(), vc.clone()
        for ab in (None, alibi):
            got = ops.ragged_attention(q, kc, vc, ss, cl, D ** -0.5, mc, ab)
            ref = ragged_ref(q, kc, vc, ss.cpu(), cl.cpu(), D ** -0.5, ab)
            name = f"ragged D{D} max_ctx {mc}{' hard' if hard else ''}{' alibi' if ab is not None else ''}"
            ck.bf16(f"ragged_attention D{D}", name, got, ref, _bf(ref))
            pad = cl == 0
            ck.require(bool((got[pad] == 0).all()), f"{name}: padding tokens are not exactly zero")
        ck.require(torch.equal(kc.view(torch.int16), bk.view(torch.int16)) and
                   torch.equal(vc.view(torch.int16), bv.view(torch.int16)), f"ragged D{D}: the cache changed")
    assert max(smem) > 48 * 1024 and min(smem) <= 48 * 1024, smem
    _report(ck)


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 5])
def test_attention_cached_native(T):
    """attention_cached_: one decode token (decode_attention with kv_len = cache_len + 1) and a 5-token prompt chunk
    (the flash-attention forward over the valid rows)."""
    from alpa_b200.ops import primitives as P
    ck = Checker()
    B, h, D, S_max, n0 = 2, 8, 64, 256, 150
    scale = D ** -0.5
    g = _gen(40 + T)
    qkv = torch.randn(B, T, h, 3, D, generator=g, device="cuda").to(BF16)
    q, kn, vn = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
    fill = NAN if T == 1 else 0.0
    kbuf = torch.full((B, S_max + 3, h, D), fill, device="cuda", dtype=BF16)
    vbuf = torch.full_like(kbuf, fill)
    kbuf[:, :n0] = torch.randn(B, n0, h, D, generator=g, device="cuda").to(BF16)
    vbuf[:, :n0] = torch.randn(B, n0, h, D, generator=g, device="cuda").to(BF16)
    bk, bv = kbuf.clone(), vbuf.clone()
    cache_len = torch.tensor(n0, dtype=torch.int32, device="cuda")
    o = P.attention_cached_(q, kn, vn, kbuf[:, :S_max], vbuf[:, :S_max], cache_len, scale)
    want_k, want_v = bk.clone(), bv.clone()
    want_k[:, n0:n0 + T] = kn
    want_v[:, n0:n0 + T] = vn
    for nm, buf, want in (("k", kbuf, want_k), ("v", vbuf, want_v)):
        ck.require(torch.equal(buf.view(torch.int16), want.view(torch.int16)), f"T{T}: {nm} cache differs")
    vis = visible(T, n0 + T, True, device="cuda")
    ref, _ = attn_fwd_ref(q, want_k[:, :n0 + T], want_v[:, :n0 + T], scale, vis)
    if T == 1:
        base = _bf(ref)
    else:
        base, _ = attn_fwd_ref(q, want_k[:, :n0 + T], want_v[:, :n0 + T], scale, vis, p_round=_bf)
    ck.bf16(f"attention_cached_ T{T}", f"attention_cached_ T{T}", o, ref, base)
    _report(ck)
