"""Attention, cross-entropy, LayerNorm and the fixed-order reductions against float64 references.

Every kernel result is compared with two things computed from the same bf16 inputs:

* a float64 reference of the operation;
* a bf16 baseline: plain PyTorch (float64) that rounds only where the kernel's design rounds.  Attention forward rounds
  the unnormalised P = exp(s - rowmax) to bf16 before P.V (the row sum stays unrounded) and rounds O.  Attention
  backward rounds P and dS = P (dP - delta) to bf16 before their products, and takes delta from the bf16 O the forward
  stored.  LayerNorm and cross entropy round only their outputs.  A kernel whose inputs include another kernel's fp32
  outputs (the LayerNorm backward takes the forward's mean and rstd) is referenced from those inputs; the producing
  kernel's outputs are checked on their own.

Rules (fixed before the first GPU run; a case that breaks them is a kernel finding, not a reason to loosen them):

* bf16 outputs: the kernel's max abs error against float64 is at most RATIO x the baseline's, and so is its relative
  Frobenius error.  RATIO = 2 is the FlashAttention convention: a correct kernel differs from the baseline only by fp32
  accumulation order and by rounding ties that fall the other way, which stays well inside 2x, while any real defect
  (a lower-precision P, a misplaced tile, a wrong mask, a scaled softmax) multiplies the error many times.  The
  baseline error is floored at FLOOR_ABS_ULPS bf16 ulps of rms(ref) (max error) and at FLOOR_FRO (relative Frobenius
  error), both below what bf16 rounding of a generic tensor gives, so only exactly representable results lean on them.
  Attention gradients can cancel to zero exactly (one key: dq = dk = 0), where fp32 arithmetic and not bf16 rounding
  sets the error; there the floor is FLOOR32 = 16 eps32 of the largest sum of |summands|.
* fp32 outputs (lse, LayerNorm mean / rstd, cross-entropy stats, dgamma / dbeta, column sums, sums of squares,
  embedding gradients): each element's error is at most TOL32 * sum |terms| of that element, TOL32 = c * eps32 with
  c ~ 840.  Summing the same terms in any other fixed order moves a result by a few eps32 * sum |terms|; a missing or
  doubled CTA slot, row or chunk moves it by a whole term, orders of magnitude more at these sizes.

Every failure message prints the kernel's error, the baseline's (or the bound's) and their ratio.

The CPU tests show the rules accept the bf16 baseline and reject known-wrong results built with the same reference
functions.  The GPU tests (`-m gpu`) run the kernels at the shapes, layouts and edges where they go wrong.  The
attention forward matrix runs in two child processes, one per forward configuration (ALPA_B200_ATTN_FWD = gen4, the
128-query tile, and gen2, the 64-query tile), because the configuration is fixed per process.
"""
import json
import math
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

F64 = torch.float64
BF16 = torch.bfloat16
NEG_INF = float("-inf")

RATIO = 2.0
FLOOR_ABS_ULPS = 2          # max-error floor: two bf16 ulps of rms(ref)
FLOOR_FRO = 2.0 ** -10      # relative Frobenius floor; generic bf16 rounding gives about 2^-9.3
TOL32 = 1e-4                # c * eps32 with c ~ 840 (eps32 = 2^-23)
EPS32 = 2.0 ** -23
FLOOR32 = 16 * EPS32        # floor for results that cancel: a few fp32 ulps of their largest summands

# ---------------------------------------------------------------------------------------------------------------------
# the rules
# ---------------------------------------------------------------------------------------------------------------------


def _bf16_ulp(x: float) -> float:
    return 2.0 ** (math.floor(math.log2(x)) - 7) if x > 0 else 0.0


def bf16_rule(name, out, ref, base, terms=None):
    """[] if `out` (the kernel's bf16 result) is within RATIO x the bf16 baseline's error against the float64 `ref`,
    else one message.  `terms` (optional, same shape): sum of |summands| of each element; FLOOR32 * terms then floors
    the baseline error too, for results that cancel to (nearly) zero, where fp32 arithmetic and not bf16 rounding
    sets the error.  Returns (messages, worst ratio)."""
    out, ref, base = out.to(F64), ref.to(F64), base.to(F64)
    if out.shape != ref.shape:
        return [f"{name}: shape {tuple(out.shape)} != {tuple(ref.shape)}"], math.inf
    if not torch.isfinite(out).all():
        return [f"{name}: {int((~torch.isfinite(out)).sum())} non-finite values"], math.inf
    if ref.numel() == 0:
        return [], 0.0
    rms = ref.pow(2).mean().sqrt().item()
    nref = ref.norm().item()
    k_max = (out - ref).abs().max().item()
    b_max = (base - ref).abs().max().item()
    k_fro = (out - ref).norm().item()
    b_fro = (base - ref).norm().item()
    d_max = max(b_max, FLOOR_ABS_ULPS * _bf16_ulp(rms))
    d_fro = max(b_fro, FLOOR_FRO * nref)
    if terms is not None:
        terms = terms.to(F64)
        d_max = max(d_max, FLOOR32 * terms.abs().max().item())
        d_fro = max(d_fro, FLOOR32 * terms.norm().item())
    if d_max == 0.0:  # the reference is exactly zero: so must the kernel be
        r = 0.0 if k_max == 0.0 else math.inf
        return ([] if r == 0.0 else [f"{name}: reference is all zero, kernel max|err| {k_max:.3e}"]), r
    r_max, r_fro = k_max / d_max, k_fro / d_fro
    ratio = max(r_max, r_fro)
    if ratio <= RATIO:
        return [], ratio
    n = max(nref, 1e-300)
    return [f"{name}: max|err| kernel {k_max:.3e} baseline {b_max:.3e} ratio {r_max:.2f}; "
            f"rel-Frobenius kernel {k_fro / n:.3e} baseline {b_fro / n:.3e} ratio {r_fro:.2f} (limit {RATIO})"], ratio


def fp32_rule(name, out, ref, terms):
    """[] if |out - ref| <= TOL32 * terms elementwise (terms = sum of |summands| of each element).  Infinite reference
    values must be matched exactly.  Returns (messages, worst ratio of error to bound)."""
    out, ref, terms = out.to(F64), ref.to(F64), terms.to(F64)
    if out.shape != ref.shape:
        return [f"{name}: shape {tuple(out.shape)} != {tuple(ref.shape)}"], math.inf
    fin = torch.isfinite(ref)
    if not torch.equal(out[~fin], ref[~fin]):
        return [f"{name}: {int((out[~fin] != ref[~fin]).sum())} infinite reference values not matched"], math.inf
    if not torch.isfinite(out[fin]).all():
        return [f"{name}: {int((~torch.isfinite(out[fin])).sum())} non-finite values"], math.inf
    if not fin.any():
        return [], 0.0
    err = (out - ref)[fin].abs()
    bound = TOL32 * terms[fin]
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    i = int(r.argmax())
    ratio = r[i].item()
    if ratio <= 1.0:
        return [], ratio
    return [f"{name}: |err| {err[i].item():.3e} > bound {bound[i].item():.3e} (TOL32 * sum|terms|), ratio "
            f"{ratio:.2f}; {int((r > 1).sum())} of {r.numel()} elements out of bound"], ratio


class Checker:
    """Collects rule failures of one case and the worst ratio per (kernel, direction)."""

    def __init__(self):
        self.fails, self.worst = [], {}

    def _add(self, key, res):
        msgs, ratio = res
        self.fails += msgs
        self.worst[key] = max(self.worst.get(key, 0.0), ratio)

    def bf16(self, key, name, out, ref, base, terms=None):
        self._add(key, bf16_rule(name, out, ref, base, terms))

    def fp32(self, key, name, out, ref, terms):
        self._add(key + " (fp32)", fp32_rule(name, out, ref, terms))

    def require(self, cond, msg):
        if not cond:
            self.fails.append(msg)


WORST = {}


def _report(ck: Checker):
    for k, v in ck.worst.items():
        WORST[k] = max(WORST.get(k, 0.0), v)
    assert not ck.fails, "\n".join(ck.fails)


@pytest.fixture(scope="module", autouse=True)
def _print_worst_ratios():
    yield
    if WORST:
        print("\n[kernel numerics] worst ratio of kernel error to baseline error (fp32: to the bound):")
        for k in sorted(WORST):
            print(f"  {k:40s} {WORST[k]:.3f}")


def _bf(t):
    return t.to(BF16).to(F64)


# ---------------------------------------------------------------------------------------------------------------------
# references (float64 on whatever device the inputs live on)
# ---------------------------------------------------------------------------------------------------------------------


def visible(Sq, Skv, causal, kv_len=None, device="cpu", shift_extra=0):
    """[Sq, Skv] bool: key j visible to query i iff j < L and, when causal, j <= i + (L - Sq); L = min(kv_len, Skv)."""
    L = Skv if kv_len is None else min(kv_len, Skv)
    i = torch.arange(Sq, device=device)[:, None]
    j = torch.arange(Skv, device=device)[None, :]
    vis = (j < L) & (i >= 0)
    if causal:
        vis = vis & (j <= i + (L - Sq) + shift_extra)
    return vis


def _bhsd(t):
    return t.to(F64).permute(0, 2, 1, 3)


def attn_fwd_ref(q, k, v, scale, vis, p_round=None):
    """(o [B,Sq,h,D], lse [B,h,Sq]) in float64.  p_round=None is the exact reference; otherwise the unnormalised
    P = exp(s - rowmax) goes through p_round before P.V and O is rounded to bf16 (the baseline, or a wrong variant)."""
    qf, kf, vf = _bhsd(q), _bhsd(k), _bhsd(v)
    s = (qf @ kf.transpose(-1, -2) * scale).masked_fill(~vis, NEG_INF)
    lse = torch.logsumexp(s, -1)
    m = s.amax(-1, keepdim=True)
    m = m.masked_fill(m == NEG_INF, 0.0)
    pt = torch.exp(s - m)
    den = pt.sum(-1, keepdim=True)
    den = den.masked_fill(den == 0, 1.0)
    o = ((pt if p_round is None else p_round(pt)) @ vf) / den
    o = o.permute(0, 2, 1, 3)
    return (o if p_round is None else _bf(o)), lse


def attn_bwd_ref(do, q, k, v, o, lse, scale, vis, rounded):
    """(dq, dk, dv) [B,S,h,D] in float64 given the forward's o and lse.  rounded=True rounds P and dS to bf16 before
    their products and the results to bf16 (the baseline)."""
    qf, kf, vf, dof, of = _bhsd(q), _bhsd(k), _bhsd(v), _bhsd(do), _bhsd(o)
    lse = lse.to(F64)
    s = (qf @ kf.transpose(-1, -2) * scale).masked_fill(~vis, NEG_INF)
    p = torch.exp(s - lse.masked_fill(lse == NEG_INF, 0.0)[..., None])
    r = _bf if rounded else (lambda t: t)
    dv = r(p).transpose(-1, -2) @ dof
    dp = dof @ vf.transpose(-1, -2)
    delta = (dof * of).sum(-1, keepdim=True)
    ds = r(p * (dp - delta))
    dq = ds @ kf * scale
    dk = ds.transpose(-1, -2) @ qf * scale
    return tuple(r(t.permute(0, 2, 1, 3)) for t in (dq, dk, dv))


def attn_bwd_terms(do, q, k, v, o, lse, scale, vis):
    """Sums of |summands| of dq, dk, dv (the cancellation floor of the bf16 rule): |P| (|dO| |V|^T + |delta terms|)."""
    qf, kf, vf, dof, of = (_bhsd(t).abs() for t in (q, k, v, do, o))
    lse = lse.to(F64)
    s = (_bhsd(q) @ _bhsd(k).transpose(-1, -2) * scale).masked_fill(~vis, NEG_INF)
    p = torch.exp(s - lse.masked_fill(lse == NEG_INF, 0.0)[..., None])
    dsa = p * (dof @ vf.transpose(-1, -2) + (dof * of).sum(-1, keepdim=True))
    return tuple(t.permute(0, 2, 1, 3) for t in (dsa @ kf * scale, dsa.transpose(-1, -2) @ qf * scale,
                                                   p.transpose(-1, -2) @ dof))


def ce_grad_ref(logits, labels, row_scale, vocab_start=0, gmax=None, gsum=None):
    """(softmax - onehot) * row_scale in float64 over the local shard `logits`; gmax / gsum are the global row max and
    sum of exp(x - gmax) (default: this shard is the whole vocabulary)."""
    x = logits.to(F64)
    if gmax is None:
        gmax = x.amax(1)
        gsum = torch.exp(x - gmax[:, None]).sum(1)
    p = torch.exp(x - gmax[:, None]) / gsum[:, None]
    local = labels - vocab_start
    ok = (local >= 0) & (local < x.shape[1])
    onehot = torch.zeros_like(p)
    onehot.scatter_(1, local.clamp(0, x.shape[1] - 1)[:, None], ok.to(F64)[:, None])
    return (p - onehot) * row_scale.to(F64)[:, None], ok


def check_ce_grad(ck, name, g, ref, labels, row_scale, vocab_start, full_vocab):
    """The cross-entropy gradient checks: every column under the bf16 rule (the whole tensor, and separately the
    softmax part off the label column, which the label column would otherwise dominate), zero rows exactly zero, and
    row sums ~ 0 relative to the row's L1 norm when the shard is the whole vocabulary (each element's bf16 rounding
    moves the sum by at most 2^-8 of the element)."""
    g64 = g.to(F64)
    base = _bf(ref)
    ck.bf16("ce_grad", f"{name} grad", g64, ref, base)
    local = (labels - vocab_start).clamp(0, ref.shape[1] - 1)
    off = torch.ones_like(ref, dtype=torch.bool)
    off.scatter_(1, local[:, None], False)
    ck.bf16("ce_grad", f"{name} grad off the label column", g64[off], ref[off], base[off])
    zero = row_scale == 0
    ck.require(bool((g64[zero] == 0).all()), f"{name}: rows with row_scale 0 are not exactly zero")
    if full_vocab:
        rs = g64.sum(1).abs()
        l1 = g64.abs().sum(1)
        bad = rs > 2.0 ** -8 * l1 + 8 * EPS32 * row_scale.to(F64).abs()   # bf16 rounding + fp32 error of p - 1
        ck.require(not bool(bad.any()), f"{name}: {int(bad.sum())} rows whose gradient sum exceeds 2^-8 x its L1 norm "
                                        f"(worst |sum|/L1 = {(rs / l1.clamp_min(1e-30)).max().item():.3e})")


def ln_fwd_ref(x, g, b, eps):
    """(y, mean, rstd) in float64 and the fp32-rule terms of mean and rstd."""
    xf = x.to(F64)
    H = xf.shape[-1]
    mean = xf.mean(-1)
    d = xf - mean[:, None]
    var = d.pow(2).mean(-1)
    rstd = (var + eps).rsqrt()
    y = d * rstd[:, None] * g.to(F64) + b.to(F64)
    t_mean = xf.abs().sum(-1) / H
    t_rstd = rstd * var / (var + eps)
    return y, mean, rstd, t_mean, t_rstd


def ln_bwd_ref(dy, x, g, mean, rstd):
    """(dx, dgamma, dbeta) in float64 and the terms of dgamma and dbeta."""
    xf, df = x.to(F64), dy.to(F64)
    xh = (xf - mean[:, None]) * rstd[:, None]
    gd = df * g.to(F64)
    dx = rstd[:, None] * (gd - gd.mean(-1, keepdim=True) - xh * (gd * xh).mean(-1, keepdim=True))
    return dx, (df * xh).sum(0), df.sum(0), (df * xh).abs().sum(0), df.abs().sum(0)


def ln_bwd_slot_rows(rows, H, sms):
    """Rows summed into CTA slot 0 by the LayerNorm backward (mirrors ln_bwd_warp_cfg / ln_bwd_warp_grid)."""
    cfg = {1: 1, 2: 1, 3: 1, 4: 1, 6: 2, 8: 2, 10: 2, 12: 4, 16: 4, 20: 4, 24: 8, 32: 8}
    wpr = cfg.get(H // 256, 0) if H % 256 == 0 else 0
    if wpr == 0:
        grid = min(rows, 2 * sms)
        return list(range(0, rows, grid)), grid
    gpc = 8 // wpr
    grid = (rows + gpc - 1) // gpc
    if grid > 2 * sms:
        iters = (rows + 2 * sms * gpc - 1) // (2 * sms * gpc)
        grid = (rows + iters * gpc - 1) // (iters * gpc)
    return [r for r in range(rows) if (r % (grid * gpc)) < gpc], grid


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the rules tell right from wrong
# ---------------------------------------------------------------------------------------------------------------------


def _attn_inputs(B, Sq, Skv, h, D, seed, device="cpu", kind="randn"):
    gen = torch.Generator(device=device).manual_seed(seed)

    def rn(*shape):
        return torch.randn(*shape, generator=gen, device=device, dtype=torch.float32)

    q, k, v, do = rn(B, Sq, h, D), rn(B, Skv, h, D), rn(B, Skv, h, D), rn(B, Sq, h, D)
    if kind in ("rising", "falling"):
        # every query's logit moves monotonically along the keys: with scale 1/sqrt(D) the logits span about 30, so
        # the running max rises in every KV tile ("rising") or is set by the first tile ("falling")
        q = q * 0.5
        q[..., 0] = 2.0
        ramp = torch.linspace(-7.5, 7.5, Skv, device=device) * D ** 0.5
        k = k * 0.5
        k[..., 0] = (ramp if kind == "rising" else ramp.flip(0))[None, :, None]
    elif kind == "identical":
        k = k[:, :1].expand(B, Skv, h, D).contiguous()
    return tuple(t.to(BF16) for t in (q, k, v, do))


def test_rule_accepts_baseline_and_rejects_wrong_attention():
    B, S, h, D = 1, 200, 2, 64
    q, k, v, do = _attn_inputs(B, S, S, h, D, 0)
    scale = D ** -0.5
    vis = visible(S, S, False)
    ref_o, ref_lse = attn_fwd_ref(q, k, v, scale, vis)
    base_o, _ = attn_fwd_ref(q, k, v, scale, vis, p_round=_bf)
    assert bf16_rule("baseline", base_o, ref_o, base_o)[0] == []
    e4m3 = attn_fwd_ref(q, k, v, scale, vis, p_round=lambda p: p.to(torch.float8_e4m3fn).to(F64))[0]
    msgs, ratio = bf16_rule("P in e4m3", e4m3, ref_o, base_o)
    assert msgs and ratio > 4, ratio
    v_bad = v.clone()
    v_bad[:, 64:128] = v[:, 0:64]                           # second V tile read at tile coordinate 0
    wrong_tile = attn_fwd_ref(q, k, v_bad, scale, vis, p_round=_bf)[0]
    msgs, ratio = bf16_rule("V tile", wrong_tile, ref_o, base_o)
    assert msgs and ratio > 4, ratio
    # the exact lse passes the fp32 rule; one key dropped from the sum does not
    qf, kf = _bhsd(q), _bhsd(k)
    t_lse = (qf.abs() @ kf.abs().transpose(-1, -2) * scale).amax(-1) + ref_lse.abs()
    assert fp32_rule("lse", ref_lse.float(), ref_lse, t_lse)[0] == []
    lse_drop = attn_fwd_ref(q[:, :, :, :], k[:, :S - 1], v[:, :S - 1], scale, vis[:, :S - 1])[1]
    assert fp32_rule("lse one key dropped", lse_drop.float(), ref_lse, t_lse)[0]


def test_rule_rejects_causal_mask_off_by_one_in_backward():
    B, S, h, D = 1, 128, 2, 64
    q, k, v, do = _attn_inputs(B, S, S, h, D, 1)
    scale = D ** -0.5
    vis = visible(S, S, True)
    ref_o, ref_lse = attn_fwd_ref(q, k, v, scale, vis)
    base_o, _ = attn_fwd_ref(q, k, v, scale, vis, p_round=_bf)
    ref = attn_bwd_ref(do, q, k, v, ref_o, ref_lse, scale, vis, rounded=False)
    base = attn_bwd_ref(do, q, k, v, base_o, ref_lse, scale, vis, rounded=True)
    for name, r, b in zip(("dq", "dk", "dv"), ref, base):
        assert bf16_rule(name, b, r, b)[0] == []
    wrong = attn_bwd_ref(do, q, k, v, base_o, ref_lse, scale, visible(S, S, True, shift_extra=1), rounded=True)
    rejected = [bool(bf16_rule(name, w, r, b)[0]) for name, w, r, b in zip(("dq", "dk", "dv"), wrong, ref, base)]
    assert all(rejected), rejected


def test_rule_rejects_scaled_ce_softmax():
    T, V = 64, 51200
    gen = torch.Generator().manual_seed(2)
    logits = (torch.randn(T, V, generator=gen) * 2).to(BF16)
    labels = torch.randint(0, V, (T,), generator=gen)
    labels[5] = -100
    row_scale = torch.full((T,), 1.0 / T)
    row_scale[5] = 0.0
    ref, _ = ce_grad_ref(logits, labels, row_scale)
    ck = Checker()
    check_ce_grad(ck, "baseline", _bf(ref).to(BF16), ref, labels, row_scale, 0, True)
    assert ck.fails == []
    onehot = torch.zeros(T, V, dtype=F64).scatter_(1, labels.clamp(0)[:, None], (labels >= 0).to(F64)[:, None])
    wrong = _bf(ref + onehot * row_scale.to(F64)[:, None]) * 0.9 - onehot * row_scale.to(F64)[:, None]
    ck = Checker()
    check_ce_grad(ck, "softmax x0.9", wrong.to(BF16), ref, labels, row_scale, 0, True)
    assert len(ck.fails) >= 2, ck.fails           # off-label bf16 rule and row sums


def test_rule_rejects_layernorm_dgamma_missing_a_slot():
    rows, H, sms = 4096, 256, 132
    gen = torch.Generator().manual_seed(3)
    x = (8 + torch.randn(rows, H, generator=gen)).to(BF16)
    dy = torch.randn(rows, H, generator=gen).to(BF16)
    g = torch.randn(H, generator=gen).to(BF16)
    b = torch.randn(H, generator=gen).to(BF16)
    y, mean, rstd, t_mean, t_rstd = ln_fwd_ref(x, g, b, 1e-5)
    assert bf16_rule("y", _bf(y), y, _bf(y))[0] == []
    xf = x.float()
    assert fp32_rule("mean", xf.mean(-1), mean, t_mean)[0] == []
    assert fp32_rule("rstd", torch.rsqrt(xf.var(-1, unbiased=False) + 1e-5), rstd, t_rstd)[0] == []
    dx, dg, db, t_dg, t_db = ln_bwd_ref(dy, x, g, mean, rstd)
    xh32 = ((xf - mean.float()[:, None]) * rstd.float()[:, None])
    dg32 = (dy.float() * xh32).flip(0).sum(0)             # fp32, another fixed order
    assert fp32_rule("dgamma", dg32, dg, t_dg)[0] == []
    slot_rows, slots = ln_bwd_slot_rows(rows, H, sms)
    assert slots == 256 and len(slot_rows) == 16
    keep = torch.ones(rows, dtype=torch.bool)
    keep[slot_rows] = False
    assert fp32_rule("dgamma missing slot 0", (dy.float() * xh32)[keep].sum(0), dg, t_dg)[0]
    assert fp32_rule("dbeta doubled slot 0", dy.float().sum(0) + dy.float()[slot_rows].sum(0), db, t_db)[0]


def test_rule_rejects_embedding_grad_with_a_duplicate_dropped():
    T, H, V = 2048, 64, 50
    gen = torch.Generator().manual_seed(4)
    ids = torch.randint(0, V, (T,), generator=gen)
    dy = torch.randn(T, H, generator=gen).to(BF16)
    ref = torch.zeros(V, H, dtype=F64).index_add_(0, ids, dy.to(F64))
    terms = torch.zeros(V, H, dtype=F64).index_add_(0, ids, dy.to(F64).abs())
    ok = torch.zeros(V, H).index_add_(0, ids, dy.float())
    assert fp32_rule("embedding", ok, ref, terms)[0] == []
    dup = int((ids == ids[0]).nonzero()[1])                 # the second token with the first token's id
    keep = torch.ones(T, dtype=torch.bool)
    keep[dup] = False
    wrong = torch.zeros(V, H).index_add_(0, ids[keep], dy.float()[keep])
    assert fp32_rule("embedding, one duplicate dropped", wrong, ref, terms)[0]


def test_attention_fallback_rows_without_keys():
    """The PyTorch fallback agrees with the native kernels on rows that see no key (causal, Sq > Skv): O = 0,
    lse = -inf and zero gradients, no NaN; the other rows match the float64 reference."""
    from alpa_b200.ops import primitives as P
    B, Sq, Skv, h, D = 2, 40, 24, 2, 32
    q, k, v, do = _attn_inputs(B, Sq, Skv, h, D, 5)
    scale = D ** -0.5
    o, lse = P.attention(q, k, v, scale, True)
    dq, dk, dv = P.attention_bwd(do, q, k, v, o, lse, scale, True)
    for t in (o, dq, dk, dv):
        assert torch.isfinite(t.float()).all()
    empty = Sq - Skv
    assert (o[:, :empty] == 0).all() and (dq[:, :empty] == 0).all()
    assert (lse[:, :, :empty] == NEG_INF).all() and torch.isfinite(lse[:, :, empty:]).all()
    vis = visible(Sq, Skv, True)
    ref_o, ref_lse = attn_fwd_ref(q, k, v, scale, vis)
    base_o, _ = attn_fwd_ref(q, k, v, scale, vis, p_round=_bf)
    assert bf16_rule("fallback o", o, ref_o, base_o)[0] == []
    ref = attn_bwd_ref(do, q, k, v, ref_o, ref_lse, scale, vis, rounded=False)
    base = attn_bwd_ref(do, q, k, v, base_o, ref_lse, scale, vis, rounded=True)
    for name, got, r, b in zip(("dq", "dk", "dv"), (dq, dk, dv), ref, base):
        assert bf16_rule(f"fallback {name}", got, r, b)[0] == [], name
    packed = torch.stack([q[:, :Skv], k, v], dim=3)             # [B,S,h,3,D], Sq = Skv: every row sees a key
    o2, _ = P.attention_qkvpacked(packed, scale, True)
    assert torch.isfinite(o2.float()).all()


# ---------------------------------------------------------------------------------------------------------------------
# GPU: attention
# ---------------------------------------------------------------------------------------------------------------------
HEAD_DIMS = [32, 64, 80, 96, 128]
SEQS = [1, 63, 64, 65, 127, 129, 200, 1024]


def _attn_cases():
    """(id, spec) of every attention case; spec = dict(D, Sq, Skv, causal, kind, layout, scale_mul)."""
    cases = []
    for D in HEAD_DIMS:
        for S in SEQS:
            for causal in (False, True):
                cases.append(dict(D=D, Sq=S, Skv=S, causal=causal))
        for Sq, Skv in [(64, 200), (100, 300), (300, 100)]:
            cases.append(dict(D=D, Sq=Sq, Skv=Skv, causal=True))
    for D in (64, 128):
        for causal in (False, True):
            cases.append(dict(D=D, Sq=256, Skv=256, causal=causal, scale_mul=8.0))
            for kind in ("rising", "falling", "identical"):
                cases.append(dict(D=D, Sq=256, Skv=256, causal=causal, kind=kind))
    for D in (64, 80):
        for layout in ("s3hd", "sh3d"):
            cases.append(dict(D=D, Sq=200, Skv=200, causal=True, layout=layout))
    out = []
    for c in cases:
        c.setdefault("kind", "randn")
        c.setdefault("layout", "separate")
        c.setdefault("scale_mul", 1.0)
        out.append((f"D{c['D']}-q{c['Sq']}-k{c['Skv']}-{'causal' if c['causal'] else 'full'}-{c['kind']}"
                    f"-{c['layout']}" + (f"-x{c['scale_mul']:g}" if c["scale_mul"] != 1.0 else ""), c))
    return out


ATTN_CASES = _attn_cases()


def _attn_tensors(c, seed):
    D, Sq, Skv = c["D"], c["Sq"], c["Skv"]
    h = 2
    B = 1 if max(Sq, Skv) >= 1024 else 2
    q, k, v, do = _attn_inputs(B, Sq, Skv, h, D, seed, device="cuda", kind=c["kind"])
    if c["layout"] == "s3hd":
        qkv = torch.stack([q, k, v], dim=2)                 # [B,S,3,h,D]
        q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    elif c["layout"] == "sh3d":
        qkv = torch.stack([q, k, v], dim=3)                 # [B,S,h,3,D]
        q, k, v = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
    return q, k, v, do, c["scale_mul"] * D ** -0.5


def _lse_terms(q, k, scale, vis):
    """fp32-rule terms of lse: |lse| plus scale * sum_d |q_d k_d| of the largest visible logit's products."""
    t = (_bhsd(q).abs() @ _bhsd(k).abs().transpose(-1, -2) * scale).masked_fill(~vis, 0.0)
    return t.amax(-1)


def attention_forward_case(ck, c, seed, C, kv_len=None):
    """Runs the forward kernel on case c and checks o and lse; returns the inputs, the kernel's o and lse, the mask and
    the float64 reference / bf16 baseline of the forward."""
    q, k, v, do, scale = _attn_tensors(c, seed)
    kl = None if kv_len is None else torch.tensor([kv_len], dtype=torch.int32, device="cuda")
    o, lse = C.attention_fwd(q, k, v, scale, c["causal"], kl)
    vis = visible(c["Sq"], c["Skv"], c["causal"], kv_len, device="cuda")
    ref_o, ref_lse = attn_fwd_ref(q, k, v, scale, vis)
    base_o, _ = attn_fwd_ref(q, k, v, scale, vis, p_round=_bf)
    name = f"attn fwd {c['id']}" + ("" if kv_len is None else f" kv_len={kv_len}")
    ck.require(bool(torch.isfinite(o.float()).all()), f"{name}: non-finite O")
    ck.require(not bool(lse.isnan().any()), f"{name}: NaN lse")
    empty = ~vis.any(-1)                                     # query rows that see no key: O = 0, lse = -inf
    if empty.any():
        ck.require(bool((o[:, empty] == 0).all()), f"{name}: rows without keys have O != 0")
        ck.require(bool((lse[:, :, empty] == NEG_INF).all()), f"{name}: rows without keys have lse != -inf")
    ck.bf16("attention fwd o", f"{name} o", o[:, ~empty], ref_o[:, ~empty], base_o[:, ~empty])
    ck.fp32("attention fwd lse", f"{name} lse", lse, ref_lse, ref_lse.abs() + _lse_terms(q, k, scale, vis))
    if c["kind"] == "identical" and not c["causal"]:
        mean_v = _bhsd(v).mean(-2, keepdim=True).expand(-1, -1, c["Sq"], -1).permute(0, 2, 1, 3)
        ck.bf16("attention fwd o", f"{name} O = mean(V)", o, mean_v, _bf(mean_v))
    return q, k, v, do, scale, o, lse, vis, ref_o, ref_lse, base_o


def _fwd_child_main():
    """Child process: the attention forward matrix under the configuration in ALPA_B200_ATTN_FWD."""
    from alpa_b200 import ops
    C = ops.native_module()
    torch.cuda.set_device(0)
    fails, worst = [], {}
    n = 0
    for i, (cid, c) in enumerate(ATTN_CASES):
        ck = Checker()
        attention_forward_case(ck, dict(c, id=cid), 1000 + i, C)
        fails += ck.fails
        for kk, v in ck.worst.items():
            worst[kk] = max(worst.get(kk, 0.0), v)
        n += 1
    c = dict(D=64, Sq=65, Skv=192, causal=False, kind="randn", layout="separate", scale_mul=1.0)
    for causal in (False, True):
        for L in (0, 1, 63, 64, 65, 192, 199):
            ck = Checker()
            cc = dict(c, causal=causal, id=f"D64-q65-k192-{'causal' if causal else 'full'}")
            attention_forward_case(ck, cc, 7, C, kv_len=L)
            fails += ck.fails
            for kk, v in ck.worst.items():
                worst[kk] = max(worst.get(kk, 0.0), v)
            n += 1
    torch.cuda.synchronize()
    print(json.dumps({"config": os.environ.get("ALPA_B200_ATTN_FWD", "gen4"), "cases": n, "fails": fails,
                      "worst": worst}), flush=True)
    return 0


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["gen4", "gen2"])
def test_attention_forward_matrix(config):
    """The whole forward matrix (head dims, sequence lengths, Sq != Skv, hard logits, packed layouts, kv_len) in a child
    process per forward configuration."""
    env = dict(os.environ, ALPA_B200_ATTN_FWD=config)
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "fwd-matrix"]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert r.returncode == 0 and lines, f"child exited with {r.returncode}:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    res = json.loads(lines[-1])
    print(f"\n[attention forward] configuration {res['config']}: {res['cases']} cases, worst ratios "
          + ", ".join(f"{k} {v:.3f}" for k, v in sorted(res["worst"].items())))
    assert res["config"] == config
    for k, v in res["worst"].items():
        WORST[f"{k} [{config}]"] = v
    assert not res["fails"], "\n".join(res["fails"])


@pytest.mark.gpu
@pytest.mark.parametrize("cid,c", ATTN_CASES, ids=[cid for cid, _ in ATTN_CASES])
def test_attention_backward(cid, c):
    """dq, dk, dv from the kernel's own o and lse against float64; rows without keys give zero gradients."""
    from alpa_b200 import ops
    C = ops.native_module()
    ck = Checker()
    seed = 1000 + [i for i, _ in ATTN_CASES].index(cid)      # the inputs of the same case in the forward matrix
    fwd = Checker()                                          # the forward is checked by test_attention_forward_matrix
    q, k, v, do, scale, o, lse, vis, ref_o, ref_lse, base_o = attention_forward_case(fwd, dict(c, id=cid), seed, C)
    dq, dk, dv = C.attention_bwd(do, q, k, v, o, lse, scale, c["causal"])
    ref =attn_bwd_ref(do, q, k, v, ref_o, ref_lse, scale, vis, rounded=False)
    base = attn_bwd_ref(do, q, k, v, base_o, ref_lse, scale, vis, rounded=True)
    terms = attn_bwd_terms(do, q, k, v, ref_o, ref_lse, scale, vis)
    for nm, got, r, b, t in zip(("dq", "dk", "dv"), (dq, dk, dv), ref, base, terms):
        ck.bf16(f"attention bwd {nm}", f"attn bwd {cid} {nm}", got, r, b, t)
    empty = ~vis.any(-1)
    if empty.any():
        ck.require(bool((dq[:, empty] == 0).all()), f"{cid}: rows without keys have dq != 0")
    _report(ck)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [64, 80, 128])
def test_attention_backward_into_packed_slots(D):
    """attention_qkvpacked_bwd writes dq / dk / dv into dqkv[:, :, :, i] of one [B,S,h,3,D] buffer: every element of a
    slot is written, the neighbouring slots are not touched, and the values equal the contiguous outputs bit for bit."""
    from alpa_b200 import ops
    C = ops.native_module()
    B, S, h = 2, 200, 3
    q, k, v, do = _attn_inputs(B, S, S, h, D, 11, device="cuda")
    qkv = torch.stack([q, k, v], dim=3)
    q, k, v = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
    scale = D ** -0.5
    o, lse = C.attention_fwd(q, k, v, scale, True)
    want = C.attention_bwd(do, q, k, v, o, lse, scale, True)
    full = torch.full_like(qkv, float("nan"))
    C.attention_bwd(do, q, k, v, o, lse, scale, True, full[:, :, :, 0], full[:, :, :, 1], full[:, :, :, 2])
    for i in range(3):
        assert torch.equal(full[:, :, :, i], want[i]), f"slot {i} differs from the contiguous result"
        one = torch.full_like(qkv, float("nan"))
        outs = [None, None, None]
        outs[i] = one[:, :, :, i]
        C.attention_bwd(do, q, k, v, o, lse, scale, True, *outs)
        assert torch.equal(one[:, :, :, i], want[i]), f"slot {i} written alone differs"
        others = [j for j in range(3) if j != i]
        assert one[:, :, :, others].isnan().all(), f"writing slot {i} touched a neighbouring slot"
    g = ops.attention_qkvpacked_bwd(do, qkv, o, lse, scale, True)
    assert torch.equal(g, full)


@pytest.mark.gpu
def test_attention_kv_len_ignores_rows_past_it():
    """Rows at or beyond kv_len in the cache do not change o or lse: large values there give the same bits."""
    from alpa_b200 import ops
    C = ops.native_module()
    B, Sq, Skv, h, D = 2, 65, 192, 2, 64
    for causal in (False, True):
        for L in (0, 1, 63, 64, 65, 192, 199):
            q, k, v, _ = _attn_inputs(B, Sq, Skv, h, D, 13, device="cuda")
            kl = torch.tensor([L], dtype=torch.int32, device="cuda")
            o1, l1 = C.attention_fwd(q, k, v, D ** -0.5, causal, kl)
            k2, v2 = k.clone(), v.clone()
            k2[:, L:] = 3.0e4
            v2[:, L:] = -3.0e4
            o2, l2 = C.attention_fwd(q, k2, v2, D ** -0.5, causal, kl)
            assert torch.equal(o1, o2) and torch.equal(l1, l2), f"kv_len={L} causal={causal}: cache rows past kv_len leak"


@pytest.mark.gpu
@pytest.mark.parametrize("D,causal", [(64, True), (128, False), (80, True)])
def test_attention_backward_is_reproducible(D, causal):
    from alpa_b200 import ops
    C = ops.native_module()
    q, k, v, do = _attn_inputs(2, 1024, 1024, 4, D, 17, device="cuda")
    o, lse = C.attention_fwd(q, k, v, D ** -0.5, causal)
    a = C.attention_bwd(do, q, k, v, o, lse, D ** -0.5, causal)
    b = C.attention_bwd(do, q, k, v, o, lse, D ** -0.5, causal)
    for nm, x, y in zip(("dq", "dk", "dv"), a, b):
        assert torch.equal(x, y), f"{nm} differs between two runs"


# ---------------------------------------------------------------------------------------------------------------------
# GPU: cross entropy
# ---------------------------------------------------------------------------------------------------------------------
CE_CASES = [(V, kind) for V in (8, 4104, 50272, 51200) for kind in ("randn2", "randn20", "equal")]


def _ce_inputs(T, V, kind, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "equal":
        x = torch.full((T, V), 1.5, device="cuda")
    else:
        x = torch.randn(T, V, device="cuda", generator=gen) * (2.0 if kind == "randn2" else 20.0)
    labels = torch.randint(0, V, (T,), device="cuda", generator=gen)
    labels[3::17] = -100
    row_scale = (1.0 + torch.rand(T, device="cuda", generator=gen)) / T
    row_scale[labels == -100] = 0.0
    row_scale[5::23] = 0.0                                   # masked rows with a valid label
    return x.to(BF16), labels, row_scale


def _ce_stats_check(ck, name, stats, logits, labels, vocab_start):
    x = logits.to(F64)
    mx = x.amax(1)
    e = torch.exp(x - mx[:, None])
    local = labels - vocab_start
    ok = (local >= 0) & (local < x.shape[1])
    tgt = x.gather(1, local.clamp(0, x.shape[1] - 1)[:, None])[:, 0] * ok
    ck.fp32("ce_stats", f"{name} max", stats[:, 0], mx, mx.abs())
    ck.fp32("ce_stats", f"{name} sumexp", stats[:, 1], e.sum(1), e.sum(1))
    ck.fp32("ce_stats", f"{name} target", stats[:, 2], tgt, tgt.abs())


@pytest.mark.gpu
@pytest.mark.parametrize("V,kind", CE_CASES)
def test_cross_entropy(V, kind):
    """ce_stats and ce_grad_ on a row-strided slice of a wider buffer (columns past V stay untouched), and the
    ops.cross_entropy autograd path."""
    from alpa_b200 import ops
    C = ops.native_module()
    T = 256 if V > 10000 else 512
    logits, labels, row_scale = _ce_inputs(T, V, kind, V)
    ck = Checker()
    name = f"ce V={V} {kind}"
    buf = torch.full((T, V + 72), 7.0, device="cuda", dtype=BF16)
    buf[:, :V] = logits
    view = buf[:, :V]
    stats = C.ce_stats(view, labels, 0)
    _ce_stats_check(ck, name, stats, logits, labels, 0)
    C.ce_grad_(view, labels, stats[:, :2].contiguous(), row_scale, 0)
    ck.require(bool((buf[:, V:] == 7.0).all()), f"{name}: ce_grad_ wrote past column V")
    ref, _ = ce_grad_ref(logits, labels, row_scale)
    check_ce_grad(ck, name, view, ref, labels, row_scale, 0, True)
    if kind == "equal":                                      # (1/V - onehot) * row_scale
        ck.bf16("ce_grad", f"{name} uniform", view, ref, _bf(ref))
    lg = logits.clone().requires_grad_(True)
    loss, _ = ops.cross_entropy(lg, labels)
    (loss * (row_scale * T)).sum().backward()                # dloss = row_scale * T per row
    ref2, _ = ce_grad_ref(logits, labels, row_scale * T)
    check_ce_grad(ck, f"{name} autograd", lg.grad, ref2, labels, row_scale * T, 0, True)
    _report(ck)


@pytest.mark.gpu
def test_cross_entropy_vocab_shard():
    """A vocab-parallel shard with vocab_start != 0: local stats, labels outside the shard, and the gradient from the
    global (max, sum exp) statistics."""
    from alpa_b200 import ops
    C = ops.native_module()
    T, V, vs, Vl = 384, 16416, 4104, 8208
    logits, labels, row_scale = _ce_inputs(T, V, "randn2", 99)
    shard = logits[:, vs:vs + Vl]                            # row-strided view
    ck = Checker()
    stats = C.ce_stats(shard, labels, vs)
    _ce_stats_check(ck, "ce shard", stats, shard, labels, vs)
    inside = (labels >= vs) & (labels < vs + Vl)
    assert inside.any() and (~inside & (labels >= 0)).any()
    x = logits.to(F64)
    gmax = x.amax(1)
    gsum = torch.exp(x - gmax[:, None]).sum(1)
    g = shard.clone()
    C.ce_grad_(g, labels, torch.stack([gmax, gsum], 1).float(), row_scale, vs)
    ref, _ = ce_grad_ref(shard, labels, row_scale, vs, gmax, gsum)
    check_ce_grad(ck, "ce shard", g, ref, labels, row_scale, vs, False)
    _report(ck)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: LayerNorm
# ---------------------------------------------------------------------------------------------------------------------
LN_H = [256 * m for m in (1, 2, 3, 4, 6, 8, 10, 12, 16, 20, 24, 28, 32)] + [520, 1000, 2056]
_FWD_WPR = {1: 1, 2: 1, 3: 1, 4: 1, 6: 1, 8: 1, 10: 2, 12: 2, 16: 2, 20: 4, 24: 4, 28: 4, 32: 4}
_BWD_WPR = {1: 1, 2: 1, 3: 1, 4: 1, 6: 2, 8: 2, 10: 2, 12: 4, 16: 4, 20: 4, 24: 8, 32: 8}


def _ln_rows(H, sms):
    """1, 7, 9, 16384 and the row counts on either side of the switch to the balanced persistent grid (forward:
    more than 8 CTAs per SM; backward: more than 2), for the kernel that serves H."""
    fwd = _FWD_WPR.get(H // 256, 0) if H % 256 == 0 else 0
    bwd = _BWD_WPR.get(H // 256, 0) if H % 256 == 0 else 0
    f = 8 * sms * (8 // fwd if fwd else 1)
    b = 2 * sms * (8 // bwd if bwd else 1)
    return sorted({1, 7, 9, f, f + 1, b, b + 1, 16384})


def _ln_cases():
    sms = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
    return [(H, rows, res) for H in LN_H for rows in _ln_rows(H, sms) for res in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("H,rows,res", _ln_cases())
def test_layernorm(H, rows, res):
    from alpa_b200 import ops
    C = ops.native_module()
    gen = torch.Generator(device="cuda").manual_seed(H * 7 + rows)
    x = (8 + torch.randn(rows, H, device="cuda", generator=gen)).to(BF16)
    r = torch.randn(rows, H, device="cuda", generator=gen).to(BF16) if res else None
    g = (1 + 0.5 * torch.randn(H, device="cuda", generator=gen)).to(BF16)
    b = torch.randn(H, device="cuda", generator=gen).to(BF16)
    dy = torch.randn(rows, H, device="cuda", generator=gen).to(BF16)
    name = f"ln H={H} rows={rows}{' +res' if res else ''}"
    ck = Checker()
    y, mean, rstd, s = C.layernorm_fwd(x, r, g, b, 1e-5, res)
    if res:
        s_ref = x.to(F64) + r.to(F64)
        ck.bf16("layernorm fwd sum_out", f"{name} sum_out", s, s_ref, _bf(s_ref))
        xin = (x.float() + r.float()).to(BF16)               # the kernel normalises the bf16 sum it stores
    else:
        xin = x
    y_ref, m_ref, r_ref, t_mean, t_rstd = ln_fwd_ref(xin, g, b, 1e-5)
    ck.bf16("layernorm fwd y", f"{name} y", y, y_ref, _bf(y_ref))
    ck.fp32("layernorm fwd mean", f"{name} mean", mean, m_ref, t_mean)
    ck.fp32("layernorm fwd rstd", f"{name} rstd", rstd, r_ref, t_rstd)
    # the backward's inputs include the forward's fp32 mean / rstd (checked above): its reference starts from them
    dx_ref, dg_ref, db_ref, t_dg, t_db = ln_bwd_ref(dy, xin, g, mean.to(F64), rstd.to(F64))
    outs = []
    for _ in range(2):
        dg = torch.zeros(H, device="cuda")
        db = torch.zeros(H, device="cuda")
        dx = C.layernorm_bwd(dy, xin, g, mean, rstd, r, dg, db)
        outs.append((dx, dg, db))
    dx, dg, db = outs[0]
    want = dx_ref + (r.to(F64) if res else 0.0)
    ck.bf16("layernorm bwd dx" + (" + dres" if res else ""), f"{name} dx", dx, want, _bf(want))
    ck.fp32("layernorm bwd dgamma", f"{name} dgamma", dg, dg_ref, t_dg)
    ck.fp32("layernorm bwd dbeta", f"{name} dbeta", db, db_ref, t_db)
    ck.require(torch.equal(outs[0][1], outs[1][1]) and torch.equal(outs[0][2], outs[1][2]),
               f"{name}: dgamma / dbeta differ between two runs")
    ck.require(torch.equal(outs[0][0], outs[1][0]), f"{name}: dx differs between two runs")
    _report(ck)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: other fixed-order reductions
# ---------------------------------------------------------------------------------------------------------------------


def _colsum_cases():
    sms = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
    cases = []
    for N in (768, 2056):
        gy = (8 * sms + (N + 255) // 256 - 1) // ((N + 255) // 256)   # row blocks once M >= 32 * gy
        for M in sorted({1, 31, 32, 33, 32 * gy - 1, 32 * gy, 32 * gy + 1, 32 * gy * 3 + 5, 16384}):
            cases.append((M, N))
    return cases


@pytest.mark.gpu
@pytest.mark.parametrize("M,N", _colsum_cases())
def test_colsum(M, N):
    """out += column sums of a row-strided [M, N] view, around the boundaries of colsum_rows_per_block."""
    from alpa_b200 import ops
    C = ops.native_module()
    gen = torch.Generator(device="cuda").manual_seed(M + N)
    buf = torch.randn(M, N + 8, device="cuda", generator=gen).to(BF16)
    x = buf[:, :N]
    base = torch.randn(N, device="cuda", generator=gen)
    outs = []
    for _ in range(2):
        out = base.clone()
        C.colsum_(x, out)
        outs.append(out)
    ref = base.to(F64) + x.to(F64).sum(0)
    terms = base.to(F64).abs() + x.to(F64).abs().sum(0)
    ck = Checker()
    ck.fp32("colsum", f"colsum M={M} N={N}", outs[0], ref, terms)
    ck.require(torch.equal(outs[0], outs[1]), f"colsum M={M} N={N}: differs between two runs")
    _report(ck)


@pytest.mark.gpu
@pytest.mark.parametrize("extra_chunks", [0, 37])
def test_grad_sumsq(extra_chunks):
    """Sum of squares over a tensor table; extra_chunks > 0 makes more chunks than ab_sumsq_slots' CTA slots."""
    from alpa_b200 import ops
    C = ops.native_module()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    chunk = 65536
    if extra_chunks:
        sizes = [(4 * sms + extra_chunks - 3) * chunk + 12345, chunk + 1, 3 * chunk - 7]
    else:
        sizes = [1000, chunk * 2 + 3, 7]
    gen = torch.Generator(device="cuda").manual_seed(extra_chunks)
    grads = [torch.randn(n, device="cuda", generator=gen) * (i + 1) for i, n in enumerate(sizes)]
    grads[1] = grads[1].to(BF16)
    masters = [torch.zeros(n, device="cuda") for n in sizes]
    tt, cc, *_host = C.adam_build_tables(grads, masters, masters, masters, [None] * len(sizes), [0.0] * len(sizes))
    nchunks = cc.numel() // 16
    assert (nchunks > 4 * sms) == bool(extra_chunks), nchunks
    a = C.grad_sumsq(tt, cc)
    b = C.grad_sumsq(tt, cc)
    ref = sum(g.to(F64).pow(2).sum() for g in grads).reshape(1)
    ck = Checker()
    ck.fp32("grad_sumsq", f"grad_sumsq {nchunks} chunks", a, ref, ref)
    ck.require(torch.equal(a, b), "grad_sumsq differs between two runs")
    _report(ck)


@pytest.mark.gpu
@pytest.mark.parametrize("dist", ["all-equal", "zipf", "shard"])
def test_embedding_bwd(dist):
    """Scatter-add of dy rows by id with heavy duplication (all ids equal, a Zipf-like distribution) and a vocab
    shard with vocab_start != 0 and ids outside it."""
    from alpa_b200 import ops
    C = ops.native_module()
    T, H, V = 8192, 1000, 5000
    gen = torch.Generator(device="cuda").manual_seed(len(dist))
    if dist == "all-equal":
        ids = torch.full((T,), 1234, device="cuda", dtype=torch.long)
    else:
        w = 1.0 / torch.arange(1, V + 1, device="cuda", dtype=torch.float64)
        ids = torch.multinomial(w, T, replacement=True, generator=gen)
    vs, Vl = (1000, 2000) if dist == "shard" else (0, V)
    dy = torch.randn(T, H, device="cuda", generator=gen).to(BF16)
    base = torch.randn(Vl, H, device="cuda", generator=gen)
    outs = []
    for _ in range(2):
        dt = base.clone()
        C.embedding_bwd_(ids, dy, dt, vs)
        outs.append(dt)
    local = ids - vs
    ok = (local >= 0) & (local < Vl)
    ref = base.to(F64).index_add(0, local[ok], dy.to(F64)[ok])
    terms = base.to(F64).abs().index_add(0, local[ok], dy.to(F64)[ok].abs())
    ck = Checker()
    ck.fp32("embedding_bwd", f"embedding_bwd {dist}", outs[0], ref, terms)
    ck.require(torch.equal(outs[0], outs[1]), f"embedding_bwd {dist}: differs between two runs")
    _report(ck)


if __name__ == "__main__":
    if sys.argv[1:] == ["fwd-matrix"]:
        sys.exit(_fwd_child_main())
    sys.exit(f"usage: {sys.argv[0]} fwd-matrix")
