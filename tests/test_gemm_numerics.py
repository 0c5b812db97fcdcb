"""The bf16, fp8 and MXFP8 GEMMs, their epilogues, the quantisers and the decode GEMV against float64 references.

Every reference is float64 and is computed from the exact bf16 / e4m3 values the kernel read.  The bf16 baseline rounds
only where the kernel's design rounds: the bf16 output once; `aux_out`, the pre-activation, to bf16 (the activation
itself is applied to the unrounded value); bf16 `accumulate` as bf16(old + result).  The decode GEMV's LayerNorm
prologue rounds its output to bf16, and with fp8 weights it quantises each token to e4m3; the reference quantises with
the same fp32 formula and takes the result as the kernel's input.

Rules (fixed before the first GPU run; a case that breaks them is a kernel finding, never a reason to loosen them):

* bf16 outputs: `bf16_rule` of tests/test_kernel_numerics.py (max error and relative Frobenius error at most RATIO = 2
  times the baseline's).
* fp32 outputs (`out_fp32`, fp32 `accumulate`): |err| <= max(TOL32, 2 ceil(K / 16) eps32) * sum|terms| per element,
  sum|terms| = sum_k |alpha a_ik b_kj| + |bias| + |residual| + |old|.  That allows one fp32 rounding per wgmma k-step
  with a factor of 2 to spare.  These cases use positive-mean operands, so a dropped or doubled 64-wide k-block moves an
  element by about 64 / K of sum|terms|: 16x the bound at K = 16384.
* Quantisers: MXFP8 `q` and scale atoms bit-exact against `primitives._quantize_mxfp8_ref`, padding bytes included.
  Per-row e4m3: the scale equals fp32(max(amax, 1e-8) * fp32(1 / 448)) bit for bit, and `q` equals round-to-nearest-
  even of x / scale, except where x / scale lies within MIDPOINT_ULPS fp32 ulps of an e4m3 rounding midpoint (the
  kernel multiplies by an approximate 1 / scale); there either neighbour passes.  A result more than one e4m3 step off
  always fails.

The CPU tests show the rules accept each baseline and reject wrong results built with the same reference code.  The
GPU tests (`-m gpu`) call the bindings at the shapes, layouts and edges where these kernels go wrong: tails, partial and
many k-blocks, both tile widths and all operand majors, batches with padded batch strides, operands inside NaN-filled
buffers (a read outside the matrix poisons the result) and outputs inside sentinel-filled buffers (a write outside
the view changes the sentinel).
"""
import itertools
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernel_numerics import (EPS32, TOL32, Checker, attn_fwd_ref, bf16_rule, fp32_rule, ln_fwd_ref,  # noqa: E402
                                  visible)

F64 = torch.float64
BF16 = torch.bfloat16
E4M3 = torch.float8_e4m3fn
NAN = float("nan")

FP32_STEP_ULPS = 2          # fp32 outputs: roundings allowed per wgmma k-step (16 deep)
MIDPOINT_ULPS = 4           # e4m3 quantiser: fp32 ulps around a rounding midpoint where either neighbour passes
INV448 = torch.tensor(1.0 / 448.0, dtype=torch.float32).item()   # fp32(1 / 448)

ACT_NONE, ACT_GELU, ACT_RELU, ACT_DGELU, ACT_DRELU = 0, 1, 2, 3, 4

# ---------------------------------------------------------------------------------------------------------------------
# rules and the worst-ratio report
# ---------------------------------------------------------------------------------------------------------------------


def fp32_gemm_coef(K):
    return max(TOL32, FP32_STEP_ULPS * math.ceil(K / 16) * EPS32)


def gemm_fp32_rule(name, out, ref, terms, K):
    """fp32_rule with the GEMM bound max(TOL32, 2 ceil(K/16) eps32) * sum|terms|."""
    return fp32_rule(name, out, ref, terms * (fp32_gemm_coef(K) / TOL32))


def _bf(t):
    return t.to(BF16).to(F64)


def e4m3_rne(t):
    """(nearest e4m3 value of the float64 t, round-to-nearest-even, saturating at 448; the e4m3 values below and above
    |t|; whether t lies within MIDPOINT_ULPS fp32 ulps of the midpoint between them)."""
    a = t.abs()
    _, ex = torch.frexp(a)
    e = (ex.to(F64) - 1).clamp_min(-6)                     # e4m3: exponents >= -6, subnormal step 2^-9
    ulp = torch.exp2(e - 3)
    n = torch.floor(a / ulp)
    lo, hi = n * ulp, (n + 1) * ulp
    frac = a / ulp - n
    up = (frac > 0.5) | ((frac == 0.5) & (torch.remainder(n, 2) == 1))
    r = torch.where(up, hi, lo).clamp_max(448.0)
    ulp32 = torch.exp2(ex.to(F64) - 1 - 23)
    near = (a - (lo + ulp / 2)).abs() <= MIDPOINT_ULPS * ulp32
    s = torch.sign(t)
    return s * r, s * lo.clamp_max(448.0), s * hi.clamp_max(448.0), near


def e4m3_rule(name, q, sx, x):
    """Per-row e4m3 quantiser: sx bit-exact, q = RNE(x / sx) outside the midpoint windows.  Returns (messages, number
    of elements that used the midpoint exception)."""
    x32 = x.float()
    amax = x32.abs().amax(1)
    want = amax.clamp_min(1e-8) * torch.tensor(INV448, dtype=torch.float32, device=x.device)
    msgs = []
    if not torch.equal(sx.view(torch.int32), want.view(torch.int32)):
        bad = int((sx.view(torch.int32) != want.view(torch.int32)).sum())
        msgs.append(f"{name}: {bad} of {sx.numel()} row scales differ from fp32(max(amax, 1e-8) * fp32(1/448))")
        return msgs, 0
    t = x32.to(F64) / sx.to(F64)[:, None]
    r, lo, hi, near = e4m3_rne(t)
    qf = q.to(F64)
    exact = qf == r
    neighbour = near & ((qf == lo) | (qf == hi))
    bad = ~(exact | neighbour)
    if bad.any():
        i = int(bad.flatten().nonzero()[0])
        msgs.append(f"{name}: {int(bad.sum())} of {q.numel()} e4m3 values are not round-to-nearest-even of x / scale "
                    f"(first: x/scale {t.flatten()[i].item():.9g}, q {qf.flatten()[i].item()}, want {r.flatten()[i].item()})")
    return msgs, int((~exact & neighbour).sum())


WORST = {}
COUNTS = {}


def _report(ck: Checker):
    for k, v in ck.worst.items():
        WORST[k] = max(WORST.get(k, 0.0), v)
    assert not ck.fails, "\n".join(ck.fails)


@pytest.fixture(scope="module", autouse=True)
def _print_worst_ratios():
    yield
    if WORST:
        print("\n[gemm numerics] worst ratio of kernel error to baseline error (fp32: to the bound):")
        for k in sorted(WORST):
            print(f"  {k:48s} {WORST[k]:.3f}")
    for k in sorted(COUNTS):
        print(f"  {k}: {COUNTS[k]}")


# ---------------------------------------------------------------------------------------------------------------------
# references (float64 on whatever device the inputs live on)
# ---------------------------------------------------------------------------------------------------------------------


def gelu64(z):
    return 0.5 * z * (1.0 + torch.erf(z * 0.7071067811865476))


def dgelu64(z):
    return 0.5 * (1.0 + torch.erf(z * 0.7071067811865476)) + z * 0.3989422804014327 * torch.exp(-0.5 * z * z)


def epilogue_ref(acc, alpha=1.0, bias=None, act=ACT_NONE, aux_in=None, residual=None, old=None, fp32_out=False,
                 wrong=None):
    """The epilogue in float64 from the exact product `acc` [.., M, N].  Returns (out_ref, out_base, aux_ref,
    aux_base, terms_extra): the baseline rounds only where the kernel's design rounds.  `wrong` builds a known-wrong
    variant: alpha_after_bias, residual_before_act, aux_after_act, dgelu_at_output, drelu_ge, acc_ignores_old."""
    b = 0.0 if bias is None else bias.to(F64)
    z = acc * alpha + b if wrong != "alpha_after_bias" else (acc + b) * alpha
    r = None if residual is None else residual.to(F64)
    v = z
    if wrong == "residual_before_act" and r is not None:
        v = v + r
    if act == ACT_GELU:
        v = gelu64(v)
    elif act == ACT_RELU:
        v = v.clamp_min(0.0)
    elif act == ACT_DGELU:
        zi = aux_in.to(F64)
        v = v * (dgelu64(_bf(gelu64(zi))) if wrong == "dgelu_at_output" else dgelu64(zi))
    elif act == ACT_DRELU:
        zi = aux_in.to(F64)
        v = torch.where(zi >= 0 if wrong == "drelu_ge" else zi > 0, v, torch.zeros_like(v))
    aux_ref = z
    aux_base = _bf(v) if wrong == "aux_after_act" else _bf(z)
    if r is not None and wrong != "residual_before_act":
        v = v + r
    if old is not None and wrong != "acc_ignores_old":
        v = v + old.to(F64)
    extra = b.abs() if bias is not None else 0.0
    if r is not None:
        extra = extra + r.abs()
    if old is not None:
        extra = extra + old.to(F64).abs()
    return v, (v if fp32_out else _bf(v)), aux_ref, aux_base, extra


def gemv_ref(x, w, w_scale=None, bias=None, act=ACT_NONE, residual=None, ln=None):
    """Decode GEMV in float64: (ref, base).  fp8 weights (w_scale given): the token rows (after the LayerNorm, rounded
    to bf16) are quantised per row with the kernel's fp32 formula and rounded to nearest even; that e4m3 input is the
    reference's input.  bf16 weights: the reference uses the exact LayerNorm, the baseline rounds it to bf16."""
    xf = x.to(F64)
    if ln is not None:
        g, b, eps = ln
        mean = xf.mean(-1, keepdim=True)
        d = xf - mean
        xf = d * (d.pow(2).mean(-1, keepdim=True) + eps).rsqrt() * g.to(F64) + b.to(F64)
    if w_scale is not None:
        xr = _bf(xf).float()
        sc = xr.abs().amax(1).clamp_min(1e-8) * torch.tensor(INV448, dtype=torch.float32, device=x.device)
        xq = e4m3_rne(xr.to(F64) / sc.to(F64)[:, None])[0] * sc.to(F64)[:, None]
        x_ref = x_base = xq
        wf = w.to(F64) * w_scale.to(F64)[:, None]
    else:
        x_ref, x_base = xf, (_bf(xf) if ln is not None else xf)
        wf = w.to(F64)
    out = []
    for xi in (x_ref, x_base):
        y = xi @ wf.t()
        if bias is not None:
            y = y + bias.to(F64)
        y = gelu64(y) if act == ACT_GELU else (y.clamp_min(0.0) if act == ACT_RELU else y)
        if residual is not None:
            y = y + residual.to(F64)
        out.append(y)
    return out[0], _bf(out[1])


def mx_dequant64(q, sf):
    """float64 values of a block-scaled operand (q e4m3 [rows, K], scale atoms)."""
    from alpa_b200.ops import primitives as P
    rows, K = q.shape
    e = P.mx_unpack_scale_atoms(sf, rows, K).to(F64) - 127.0
    return (q.to(F64).view(rows, K // 32, 32) * torch.exp2(e)[..., None]).view(rows, K)


def act64(y, act):
    return gelu64(y) if act == ACT_GELU else (y.clamp_min(0.0) if act == ACT_RELU else y)


def _gen(seed, device):
    return torch.Generator(device=device).manual_seed(seed)


def mx_operand(rows, K, gen, device):
    """Values whose 32-wide K blocks and 128-row groups differ in magnitude, so that a scale taken from the wrong
    block or row group is off by a power of two."""
    x = torch.randn(rows, K, generator=gen, device=device)
    kb = torch.arange(K // 32, device=device).repeat_interleave(32)
    rg = torch.arange(rows, device=device) // 128
    return (x * torch.exp2(((kb % 5) - 2).float())[None, :] * torch.exp2((rg % 3).float())[:, None]).to(BF16)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the rules tell right from wrong
# ---------------------------------------------------------------------------------------------------------------------


def _ab(M, N, K, seed, mean=0.0, batch=None):
    g = _gen(seed, "cpu")
    lead = () if batch is None else (batch,)
    a = (torch.randn(*lead, M, K, generator=g) + mean).to(BF16)
    b = (torch.randn(*lead, K, N, generator=g) / K ** 0.5 + mean).to(BF16)
    return a, b


def test_rules_accept_baselines_and_reject_mainloop_defects():
    M, N, K = 130, 1000, 2048
    a, b = _ab(M, N, K, 0)
    ref = a.to(F64) @ b.to(F64)
    base = _bf(ref)
    assert bf16_rule("baseline", base, ref, base)[0] == []
    drop = a.clone()
    drop[:, 640:704] = 0                                    # k-block 10 of 64 never accumulated
    msgs, ratio = bf16_rule("dropped k-block", _bf(drop.to(F64) @ b.to(F64)), ref, base)
    assert msgs and ratio > 4, ratio
    twice = ref + a[:, 640:704].to(F64) @ b[640:704].to(F64)
    msgs, ratio = bf16_rule("k-block twice", _bf(twice), ref, base)
    assert msgs and ratio > 4, ratio
    shifted = base.clone()
    shifted[:, 904:] = base[:, 896:992]                     # 128-wide N tail tile written 8 columns to the right
    msgs, ratio = bf16_rule("N tail shifted", shifted, ref, base)
    assert msgs and ratio > 4, ratio


def test_fp32_rule_rejects_a_dropped_k_block_at_16384():
    M, N, K = 64, 72, 16384
    a, b = _ab(M, N, K, 1, mean=1.0)
    af, bf = a.to(F64), b.to(F64)
    ref = af @ bf
    terms = af.abs() @ bf.abs()
    assert gemm_fp32_rule("fp32 out", ref.float(), ref, terms, K)[0] == []
    # fp32 summation in 16-deep chunks (the wgmma k-step), the rounding the bound allows for
    chunks = (a.float().view(M, K // 16, 16).permute(1, 0, 2) @ b.float().view(K // 16, 16, N))
    acc = torch.zeros(M, N)
    for c in chunks:
        acc = acc + c
    msgs, ratio = gemm_fp32_rule("fp32 chunked", acc, ref, terms, K)
    assert msgs == [], msgs
    drop = ref - af[:, 4096:4160] @ bf[4096:4160]
    msgs, ratio = gemm_fp32_rule("dropped k-block", drop.float(), ref, terms, K)
    assert msgs and ratio > 8, ratio
    twice = ref + af[:, 4096:4160] @ bf[4096:4160]
    assert gemm_fp32_rule("k-block twice", twice.float(), ref, terms, K)[0]


@pytest.mark.parametrize("case,wrong", [
    ("bias_alpha", "alpha_after_bias"),
    ("bias_gelu_residual", "residual_before_act"),
    ("bias_gelu_aux", "aux_after_act"),
    ("dgelu", "dgelu_at_output"),
    ("drelu", "drelu_ge"),
    ("acc_fp32", "acc_ignores_old"),
])
def test_rules_reject_wrong_epilogues(case, wrong):
    M, N, K = 200, 136, 264
    a, b = _ab(M, N, K, 2, mean=1.0 if case == "acc_fp32" else 0.0)
    g = _gen(3, "cpu")
    acc = a.to(F64) @ b.to(F64)
    kw = {}
    if case == "bias_alpha":
        kw = dict(alpha=0.37, bias=(torch.randn(N, generator=g) * 4).to(BF16))
    elif case == "bias_gelu_residual":
        kw = dict(bias=torch.randn(N, generator=g).to(BF16), act=ACT_GELU,
                  residual=torch.randn(M, N, generator=g).to(BF16))
    elif case == "bias_gelu_aux":
        kw = dict(bias=torch.randn(N, generator=g).to(BF16), act=ACT_GELU)
    elif case in ("dgelu", "drelu"):
        kw = dict(act=ACT_DGELU if case == "dgelu" else ACT_DRELU, aux_in=aux_in_values(M, N, g, "cpu"))
    else:
        kw = dict(old=accumulate_old(M, N, K, g, "cpu", torch.float32), fp32_out=True)
    ref, base, aux_ref, aux_base, extra = epilogue_ref(acc, **kw)
    wr, wb, _, wrong_aux, _ = epilogue_ref(acc, wrong=wrong, **kw)
    if case == "acc_fp32":
        terms = a.to(F64).abs() @ b.to(F64).abs() + extra
        assert gemm_fp32_rule("baseline", base.float(), ref, terms, K)[0] == []
        assert gemm_fp32_rule(wrong, wb.float(), ref, terms, K)[0]
        return
    assert bf16_rule("baseline", base, ref, base)[0] == []
    assert bf16_rule("baseline aux", aux_base, aux_ref, aux_base)[0] == []
    if wrong == "aux_after_act":
        msgs, ratio = bf16_rule(wrong, wrong_aux, aux_ref, aux_base)
    else:
        msgs, ratio = bf16_rule(wrong, wb, ref, base)
    assert msgs and ratio > 2, ratio


def test_quantiser_rules_reject_wrong_mxfp8_scales():
    from alpa_b200.ops import primitives as P
    M, K = 300, 224                                          # partial row group, K % 128 == 96
    x = mx_operand(M, K, _gen(4, "cpu"), "cpu")
    q, sf = P._quantize_mxfp8_ref(x)
    e = P.mx_unpack_scale_atoms(sf, M, K)
    assert torch.equal(P.mx_pack_scale_atoms(e), sf)
    nb_k = P.mx_pack_scale_atoms(torch.roll(e, 1, dims=1))  # scale of the neighbouring K block
    nb_r = P.mx_pack_scale_atoms(torch.roll(e, 128, dims=0))  # scale of the neighbouring 128-row group
    assert not torch.equal(nb_k, sf) and not torch.equal(nb_r, sf)
    # the GEMM built from those scales fails the bf16 rule
    w = mx_operand(72, K, _gen(5, "cpu"), "cpu")
    wq, wsf = P._quantize_mxfp8_ref(w)
    wd = mx_dequant64(wq, wsf)
    ref = mx_dequant64(q, sf) @ wd.t()
    base = _bf(ref)
    assert bf16_rule("baseline", base, ref, base)[0] == []
    for name, bad in (("neighbouring K block", nb_k), ("neighbouring row group", nb_r)):
        msgs, ratio = bf16_rule(name, _bf(mx_dequant64(q, bad) @ wd.t()), ref, base)
        assert msgs and ratio > 2, (name, ratio)


def test_e4m3_rule_accepts_rne_and_rejects_one_step_off():
    g = _gen(6, "cpu")
    x = (torch.randn(16, 528, generator=g) * 0.7).to(BF16)
    x[3] = 0
    x[4, 17] = 900.0
    sx = x.float().abs().amax(1).clamp_min(1e-8) * torch.tensor(INV448, dtype=torch.float32)
    q = e4m3_rne(x.float().to(F64) / sx.to(F64)[:, None])[0].float().to(E4M3)
    msgs, _ = e4m3_rule("rne", q, sx, x)
    assert msgs == [], msgs
    # torch's own fp32 -> e4m3 conversion of fl32(x * fl32(1 / s)) lies inside the rule
    inv = 1.0 / sx
    assert e4m3_rule("fp32 product", (x.float() * inv[:, None]).to(E4M3), sx, x)[0] == []
    off = q.float().clone()
    off[5, 9] = e4m3_rne(off[5, 9:10].to(F64) * 1.13)[0].float()[0]      # one element one step up
    assert e4m3_rule("one step off", off.to(E4M3), sx, x)[0]
    assert e4m3_rule("scale off", q, sx * (1 + 2 ** -23), x)[0]


def test_bf16_rule_rejects_a_14_bit_fp8_accumulator_at_k_10240():
    """Hopper's fp8 wgmma keeps fewer accumulator bits than fp32.  An accumulator truncated to 14 bits after every
    32-deep step, over all of K = 10240 in one chain, breaks the bf16 rule on the fp8 serving GEMM's operand
    distribution; the same truncation with the sum promoted to fp32 every 128 K passes."""
    M, N, K = 48, 64, 10240
    g = _gen(7, "cpu")
    x = (torch.randn(M, K, generator=g) * 0.7).to(BF16)
    w = torch.randn(N, K, generator=g) * 0.05
    sw = w.abs().amax(1).clamp_min(1e-8) / 448.0
    wq = (w / sw[:, None]).to(E4M3)
    sx = x.float().abs().amax(1).clamp_min(1e-8) * torch.tensor(INV448, dtype=torch.float32)
    xq = e4m3_rne(x.float().to(F64) / sx.to(F64)[:, None])[0]
    parts = torch.einsum("msk,nsk->mns", xq.view(M, K // 32, 32), wq.to(F64).view(N, K // 32, 32))
    scale = sx.to(F64)[:, None] * sw.to(F64)[None, :]
    ref = parts.sum(-1) * scale
    base = _bf(ref)
    assert bf16_rule("baseline", base, ref, base)[0] == []

    def trunc14(v):
        m, e = torch.frexp(v)
        return torch.ldexp(torch.trunc(m * 2.0 ** 14) / 2.0 ** 14, e.to(F64))

    def chain(steps_per_promotion):
        total = torch.zeros(M, N, dtype=F64)
        acc = torch.zeros(M, N, dtype=F64)
        for s in range(K // 32):
            acc = trunc14(acc + parts[..., s])
            if (s + 1) % steps_per_promotion == 0:
                total, acc = (total + acc).float().to(F64), torch.zeros_like(acc)
        return total + acc

    msgs, ratio = bf16_rule("14-bit accumulator, one chain", _bf(chain(K // 32) * scale), ref, base)
    assert msgs and ratio > 2, ratio
    msgs, ratio = bf16_rule("14-bit accumulator, promoted every 128 K", _bf(chain(4) * scale), ref, base)
    assert msgs == [], msgs


def test_rule_rejects_swapped_gemv_tokens():
    g = _gen(8, "cpu")
    M, N, K = 5, 1000, 256
    x = torch.randn(M, K, generator=g).to(BF16)
    w = (torch.randn(N, K, generator=g) * 0.05).to(BF16)
    ref, base = gemv_ref(x, w)
    assert bf16_rule("baseline", base, ref, base)[0] == []
    swapped = base.clone()
    swapped[[1, 2]] = base[[2, 1]]
    assert bf16_rule("tokens 1 and 2 swapped", swapped, ref, base)[0]
    sw = w.float().abs().amax(1) / 448.0
    wq = (w.float() / sw[:, None]).to(E4M3)
    ref, base = gemv_ref(x, wq, sw, act=ACT_GELU)
    assert bf16_rule("fp8 baseline", base, ref, base)[0] == []
    swapped = base.clone()
    swapped[[0, 4]] = base[[4, 0]]
    assert bf16_rule("fp8 tokens 0 and 4 swapped", swapped, ref, base)[0]


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers: operands inside NaN-filled buffers, outputs inside sentinel-filled buffers
# ---------------------------------------------------------------------------------------------------------------------


def _r8(n):
    return (n + 7) // 8 * 8


def padded(values, pad_rows=3, pad_cols=8, fill=NAN):
    """`values` [.., R, C] copied into a larger buffer filled with `fill`: row stride _r8(C) + pad_cols, pad_rows extra
    rows per batch (so the batch stride is not R * ld).  Returns the view."""
    lead = values.shape[:-2]
    R, C = values.shape[-2:]
    buf = torch.full((*lead, R + pad_rows, _r8(C) + pad_cols), fill, device=values.device, dtype=values.dtype)
    view = buf[..., :R, :C]
    view.copy_(values)
    return view


class Sentinel:
    """A [.., R, C] view at row 1, column 8 of a buffer filled with NaN (bitwise pattern kept for the check)."""

    def __init__(self, shape, dtype, inside=None):
        lead = shape[:-2]
        R, C = shape[-2:]
        self.buf = torch.full((*lead, R + 2, C + 16), NAN, device="cuda", dtype=dtype)
        self.view = self.buf[..., 1:R + 1, 8:8 + C]
        if inside is not None:
            self.view.copy_(inside)
        self.before = self.buf.clone()

    def untouched_outside(self):
        mask = torch.ones_like(self.buf, dtype=torch.bool)
        mask[..., 1:self.view.shape[-2] + 1, 8:8 + self.view.shape[-1]] = False
        bits = torch.int16 if self.buf.dtype == BF16 else torch.int32
        return torch.equal(self.buf.view(bits)[mask], self.before.view(bits)[mask])


def aux_in_values(M, N, g, device, batch=None):
    """Saved pre-activations for dGELU / dReLU: randn, with exact zeros and plenty of negatives."""
    lead = () if batch is None else (batch,)
    z = torch.randn(*lead, M, N, generator=g, device=device) * 1.5
    z.view(-1)[::7] = 0.0
    return z.to(BF16)


def accumulate_old(M, N, K, g, device, dtype, batch=None):
    """Existing contents of an accumulated output (a previous partial sum of the same size as the new one)."""
    lead = () if batch is None else (batch,)
    return ((torch.rand(*lead, M, N, generator=g, device=device) + 0.5) * K).to(dtype)


def _operands_gpu(M, N, K, ta, tb, seed, batch=None, mean=0.0):
    """Logical A [.., M, K], B [.., K, N] (float64) and the stored operands as padded views in the requested majors."""
    g = _gen(seed, "cuda")
    lead = () if batch is None else (batch,)
    a = (torch.randn(*lead, M, K, generator=g, device="cuda") + mean).to(BF16)
    b = (torch.randn(*lead, K, N, generator=g, device="cuda") / (K ** 0.5 if mean == 0.0 else 1.0) + mean).to(BF16)
    sa = padded(a.transpose(-1, -2) if ta else a)           # MN-major A is stored [K, M]
    sb = padded(b if tb else b.transpose(-1, -2))            # MN-major B is stored [K, N]
    return a.to(F64), b.to(F64), sa, sb


def _native():
    from alpa_b200 import ops
    return ops.native_module()


# ---------------------------------------------------------------------------------------------------------------------
# GPU: bf16 GEMM mainloop
# ---------------------------------------------------------------------------------------------------------------------
MAINLOOP_M = [1, 127, 129, 2104]
MAINLOOP_N = [8, 72, 136, 1000, 2048]
MAINLOOP_K = [8, 16, 72, 264, 2048]
INSTANTIATIONS = [(bn, ta, tb) for bn in (128, 256) for ta in (False, True) for tb in (False, True)]


def _inst_id(bn, ta, tb):
    return f"bn{bn}-A{'mn' if ta else 'k'}-B{'mn' if tb else 'k'}"


@pytest.mark.gpu
@pytest.mark.parametrize("bn,ta,tb", INSTANTIATIONS, ids=[_inst_id(*i) for i in INSTANTIATIONS])
def test_bf16_gemm_mainloop(bn, ta, tb):
    """Every M x N x K of the grid on one instantiation: operands inside NaN buffers, output inside a NaN sentinel."""
    C = _native()
    ck = Checker()
    key = f"gemm bf16 mainloop {_inst_id(bn, ta, tb)}"
    seed = 0
    for M in MAINLOOP_M:
        for N in MAINLOOP_N:
            for K in MAINLOOP_K:
                seed += 1
                a, b, sa, sb = _operands_gpu(M, N, K, ta, tb, seed)
                out = Sentinel((M, N), BF16)
                C.gemm(sa, sb, ta, tb, out=out.view, block_n=bn)
                ref = a @ b
                name = f"{key} M{M} N{N} K{K}"
                ck.bf16(key, name, out.view, ref, _bf(ref))
                ck.require(out.untouched_outside(), f"{name}: wrote outside the output view")
    _report(ck)


@pytest.mark.gpu
@pytest.mark.parametrize("bn", [128, 256])
def test_bf16_gemm_batched_padded_strides(bn):
    C = _native()
    ck = Checker()
    for i, (ta, tb) in enumerate([(False, False), (False, True), (True, False), (True, True)]):
        M, N, K = 200, 136, 264
        a, b, sa, sb = _operands_gpu(M, N, K, ta, tb, 100 + i, batch=3)
        assert sa.stride(0) != sa.shape[1] * sa.stride(1)
        out = Sentinel((3, M, N), BF16)
        C.gemm(sa, sb, ta, tb, out=out.view, block_n=bn)
        ref = a @ b
        key = f"gemm bf16 batched bn{bn}"
        ck.bf16(key, f"{key} ta={ta} tb={tb}", out.view, ref, _bf(ref))
        ck.require(out.untouched_outside(), f"{key} ta={ta} tb={tb}: wrote outside the output view")
    _report(ck)


@pytest.mark.gpu
@pytest.mark.parametrize("M,N", [(512, 512), (136, 72), (1, 8)])
def test_bf16_gemm_wgrad_k16384(M, N):
    """dW = dY^T X at the step's token count: both operands MN-major, K = 16384, fp32 and bf16 outputs."""
    C = _native()
    ck = Checker()
    K = 16384
    a, b, sa, sb = _operands_gpu(M, N, K, True, True, 200 + M, mean=1.0)
    ref = a @ b
    terms = a.abs() @ b.abs()
    for bn in (128, 256):
        out = Sentinel((M, N), torch.float32)
        C.gemm(sa, sb, True, True, out=out.view, block_n=bn)
        key = f"gemm wgrad K16384 bn{bn}"
        ck._add(key + " (fp32)", gemm_fp32_rule(f"{key} M{M} N{N} fp32", out.view, ref, terms, K))
        ck.require(out.untouched_outside(), f"{key}: wrote outside the fp32 output view")
        o16 = Sentinel((M, N), BF16)
        C.gemm(sa, sb, True, True, out=o16.view, block_n=bn)
        ck.bf16(key, f"{key} M{M} N{N} bf16", o16.view, ref, _bf(ref))
        ck.require(o16.untouched_outside(), f"{key}: wrote outside the bf16 output view")
    _report(ck)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: bf16 GEMM epilogues
# ---------------------------------------------------------------------------------------------------------------------
EPILOGUES = ["bias", "bias_gelu_aux", "bias_relu", "residual", "bias_residual", "dgelu", "drelu", "alpha_bias",
             "out_fp32", "acc_fp32", "acc_bf16", "acc_residual", "alpha_out_fp32"]
# (M, N, K, batch, trans_a, trans_b, block_n): tails on both tile widths, the dgrad layout (B MN-major), a batch
EPI_CONFIGS = [
    (129, 1000, 264, None, False, True, 128),
    (127, 1000, 264, None, False, True, 256),
    (1, 72, 16, None, False, False, 128),
    (200, 136, 72, 3, False, True, 256),
    (200, 136, 72, 3, True, False, 128),
    (2104, 1000, 2048, None, False, True, 0),
]


def _epi_id(c):
    M, N, K, batch, ta, tb, bn = c
    return f"M{M}-N{N}-K{K}" + (f"-b{batch}" if batch else "") + f"-{'mn' if ta else 'k'}{'mn' if tb else 'k'}-bn{bn}"


@pytest.mark.gpu
@pytest.mark.parametrize("epi", EPILOGUES)
@pytest.mark.parametrize("cfg", EPI_CONFIGS, ids=[_epi_id(c) for c in EPI_CONFIGS])
def test_bf16_gemm_epilogue(epi, cfg):
    C = _native()
    ck = Checker()
    M, N, K, batch, ta, tb, bn = cfg
    fp32 = epi in ("out_fp32", "acc_fp32", "acc_residual", "alpha_out_fp32")
    seed = 100 * EPI_CONFIGS.index(cfg) + EPILOGUES.index(epi)
    a, b, sa, sb = _operands_gpu(M, N, K, ta, tb, 2000 + seed, batch=batch, mean=1.0 if fp32 else 0.0)
    g = _gen(3000 + seed, "cuda")
    shape = (batch, M, N) if batch else (M, N)
    bias = (torch.randn(N, generator=g, device="cuda")).to(BF16) if "bias" in epi else None
    res = None
    if "residual" in epi:
        res = Sentinel(shape, BF16, torch.randn(shape, generator=g, device="cuda").to(BF16))
    aux_in = Sentinel(shape, BF16, aux_in_values(M, N, g, "cuda", batch)) if epi in ("dgelu", "drelu") else None
    aux_out = Sentinel(shape, BF16) if epi == "bias_gelu_aux" else None
    act = {"bias_gelu_aux": ACT_GELU, "bias_relu": ACT_RELU, "dgelu": ACT_DGELU, "drelu": ACT_DRELU}.get(epi, ACT_NONE)
    alpha = 0.37 if epi.startswith("alpha") else 1.0
    old = None
    if epi == "acc_bf16":                                    # a partial sum of the same size as this product
        old = torch.randn(shape, generator=g, device="cuda").to(BF16)
    elif epi.startswith("acc"):
        old = accumulate_old(M, N, K, g, "cuda", torch.float32, batch)
    out = Sentinel(shape, torch.float32 if fp32 else BF16, old)
    C.gemm(sa, sb, ta, tb, out=out.view, bias=bias, residual=None if res is None else res.view,
           aux_out=None if aux_out is None else aux_out.view, aux_in=None if aux_in is None else aux_in.view,
           act=act, alpha=alpha, accumulate=old is not None, block_n=bn)
    acc = a @ b
    ref, base, aux_ref, aux_base, extra = epilogue_ref(
        acc, alpha=alpha, bias=bias, act=act, aux_in=None if aux_in is None else aux_in.view,
        residual=None if res is None else res.view, old=old, fp32_out=fp32)
    key = f"gemm bf16 epilogue {epi}"
    name = f"{key} {_epi_id(cfg)}"
    if fp32:
        terms = (a.abs() @ b.abs()) * abs(alpha) + extra
        ck._add(key + " (fp32)", gemm_fp32_rule(name, out.view, ref, terms, K))
    else:
        ck.bf16(key, name, out.view, ref, base)
    if aux_out is not None:
        ck.bf16(key + " aux_out", name + " aux_out", aux_out.view, aux_ref, aux_base)
        ck.require(aux_out.untouched_outside(), f"{name}: aux_out written outside its view")
    ck.require(out.untouched_outside(), f"{name}: wrote outside the output view")
    for t, nm in ((res, "residual"), (aux_in, "aux_in")):
        if t is not None:
            ck.require(t.untouched_outside(), f"{name}: {nm} buffer changed")
    _report(ck)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: fp8 (per-row e4m3) quantiser and GEMM
# ---------------------------------------------------------------------------------------------------------------------
FP8_K = [16, 48, 528, 2560, 10240]
FP8_N = [8, 72, 2560]
FP8_M = [1, 130, 257]
# (M, N, K): every K x N of the grid with M cycling through FP8_M, then a serving shape of 16 x 80 tiles, more than
# there are SMs, so that each CTA of the persistent kernel runs several tiles
FP8_SHAPES = [(FP8_M[i % 3], N, K) for i, (K, N) in enumerate(itertools.product(FP8_K, FP8_N))]
FP8_SHAPES.append((2048, 10240, 2560))


def _fp8_x(M, K, g):
    x = torch.randn(M, K, generator=g, device="cuda") * 0.7
    if M > 2:
        x[1] = 0.0                                           # all-zero row
        x[2, K // 3] = 700.0                                 # one outlier 10^3 x the rest of its row
    return x.to(BF16)


def _fp8_w(N, K, g):
    w = torch.randn(N, K, generator=g, device="cuda") * 0.05
    sw = (w.abs().amax(1).clamp(min=1e-8) / 448.0).float()
    return (w / sw[:, None]).to(E4M3), sw


@pytest.mark.gpu
def test_e4m3_quantiser():
    C = _native()
    msgs, exceptions = [], 0
    for i, (M, K) in enumerate([(1, 16), (130, 48), (257, 528), (64, 2560), (33, 10240)]):
        x = padded(_fp8_x(M, K, _gen(300 + i, "cuda")))     # row stride > K, NaN past the row
        q, sx = C.quantize_e4m3(x)
        m, n = e4m3_rule(f"quantize_e4m3 M{M} K{K}", q, sx, x)
        msgs += m
        exceptions += n
        if M > 2:
            msgs += [] if bool((q[1].float() == 0).all()) else [f"M{M} K{K}: all-zero row not quantised to 0"]
    COUNTS["e4m3 quantiser: elements inside a midpoint window, not RNE"] = exceptions
    assert not msgs, "\n".join(msgs)


@pytest.mark.gpu
def test_fp8_gemm():
    C = _native()
    ck = Checker()
    for i, (M, N, K) in enumerate(FP8_SHAPES):
        act = (ACT_NONE, ACT_RELU, ACT_GELU)[i % 3]
        use_bias = i % 2 == 0
        g = _gen(401 + i, "cuda")
        x = _fp8_x(M, K, g)
        wq, sw = _fp8_w(N, K, g)
        bias = (torch.randn(N, generator=g, device="cuda") * 0.1).to(BF16) if use_bias else None
        q, sx = C.quantize_e4m3(x)
        y = C.gemm_fp8_q(q, sx, wq, sw, bias, act)
        ref = (q.to(F64) @ wq.to(F64).t()) * sx.to(F64)[:, None] * sw.to(F64)[None, :]
        if bias is not None:
            ref = ref + bias.to(F64)
        ref = act64(ref, act)
        key = f"gemm fp8 K{K}"
        ck.bf16(key, f"gemm fp8 M{M} N{N} K{K} act{act} bias={use_bias}", y, ref, _bf(ref))
        y2 = C.gemm_fp8(x, wq, sw, bias, act)
        ck.require(torch.equal(y, y2), f"gemm_fp8 M{M} N{N} K{K}: differs from quantize_e4m3 + gemm_fp8_q")
    _report(ck)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: MXFP8 quantiser and GEMM
# ---------------------------------------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("M,K", [(1, 32), (200, 160), (300, 224), (129, 2592), (256, 96)])
def test_mxfp8_quantiser_bit_exact(M, K):
    from alpa_b200.ops import primitives as P
    C = _native()
    g = _gen(500 + M + K, "cuda")
    x = mx_operand(M, K, g, "cuda").float()
    x[:, :32] *= torch.logspace(-3, 3, 32, device="cuda")[None, :]        # log-spaced magnitudes inside one block
    if M > 1:
        x[1, 32:64] = 0.0                                                    # an all-zero block
        x[0, 64 % K:64 % K + 32] = torch.linspace(-1, 1, 32, device="cuda") * 448.0 * 2.0 ** -5   # max exactly 448 * 2^-5
        x[0, 64 % K + 31] = 448.0 * 2.0 ** -5
    x = padded(x.to(BF16))
    q, sf = C.quantize_mxfp8(x)
    rq, rsf = P._quantize_mxfp8_ref(x.cpu())
    assert torch.equal(sf.cpu(), rsf), f"scale atoms differ in {int((sf.cpu() != rsf).sum())} bytes (padding included)"
    assert torch.equal(q.cpu().view(torch.uint8), rq.view(torch.uint8)), \
        f"{int((q.cpu().view(torch.uint8) != rq.view(torch.uint8)).sum())} e4m3 bytes differ"


# (M, N, K): every K x N of the grid with M cycling through 1, 130, 257, then 8 x 20 tiles, more than there are SMs
MX_SHAPES = [((1, 130, 257)[i % 3], N, K) for i, (K, N) in enumerate(itertools.product((32, 96, 160, 2560, 10240), (8, 72)))]
MX_SHAPES.append((1024, 2560, 2560))


@pytest.mark.gpu
def test_mxfp8_gemm():
    from alpa_b200.ops import primitives as P
    C = _native()
    ck = Checker()
    for i, (M, N, K) in enumerate(MX_SHAPES):
        act = (ACT_NONE, ACT_RELU, ACT_GELU)[i % 3]
        use_bias = i % 2 == 1
        g = _gen(601 + i, "cuda")
        x = mx_operand(M, K, g, "cuda")
        w = mx_operand(N, K, g, "cuda")
        wq, wsf = (t.cuda() for t in P._quantize_mxfp8_ref(w.cpu()))
        bias = (torch.randn(N, generator=g, device="cuda") * 0.1).to(BF16) if use_bias else None
        q, sf = C.quantize_mxfp8(x)
        y = C.gemm_mxfp8_q(q, sf, wq, wsf, bias, act)
        ref = mx_dequant64(q, sf) @ mx_dequant64(wq, wsf).t()
        if bias is not None:
            ref = ref + bias.to(F64)
        ref = act64(ref, act)
        key = f"gemm mxfp8 K{K}"
        ck.bf16(key, f"gemm mxfp8 M{M} N{N} K{K} act{act} bias={use_bias}", y, ref, _bf(ref))
    _report(ck)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: decode GEMV
# ---------------------------------------------------------------------------------------------------------------------


def _gemv_cases():
    cases = []
    for fp8 in (True, False):
        for M in range(1, 9):
            for N, K in ((24, 64), (1000, 64), (1000, 10240)):
                cases.append(dict(M=M, N=N, K=K, fp8=fp8, act=(ACT_NONE, ACT_GELU, ACT_RELU)[M % 3],
                                  bias=M % 2 == 0, res=M % 2 == 1, ln=None))
        for M in (1, 8):
            cases.append(dict(M=M, N=50272, K=2560, fp8=fp8, act=ACT_NONE, bias=False, res=False, ln=None))
        for ln in ("generic", "mean200"):
            for M in (1, 5, 8):
                cases.append(dict(M=M, N=1000, K=2560, fp8=fp8, act=ACT_GELU, bias=True, res=M == 5, ln=ln))
    return [(f"{'fp8' if c['fp8'] else 'bf16'}-M{c['M']}-N{c['N']}-K{c['K']}-act{c['act']}"
             + ("-bias" if c["bias"] else "") + ("-res" if c["res"] else "") + (f"-ln_{c['ln']}" if c["ln"] else ""),
             dict(c, seed=1000 + i)) for i, c in enumerate(cases)]


GEMV_CASES = _gemv_cases()


@pytest.mark.gpu
@pytest.mark.parametrize("cid,c", GEMV_CASES, ids=[cid for cid, _ in GEMV_CASES])
def test_gemv_decode(cid, c):
    C = _native()
    ck = Checker()
    M, N, K = c["M"], c["N"], c["K"]
    g = _gen(c["seed"], "cuda")
    x = torch.randn(M, K, generator=g, device="cuda")
    ln = None
    if c["ln"] == "mean200":
        x = x + 200.0
    elif c["ln"] == "generic":
        x = x * 3 + 0.5
    if c["ln"]:
        ln = ((1 + 0.1 * torch.randn(K, generator=g, device="cuda")).to(BF16),
              (0.1 * torch.randn(K, generator=g, device="cuda")).to(BF16), 1e-5)
    x = padded(x.to(BF16))                                    # ldx > K, NaN past the rows
    w = torch.randn(N, K, generator=g, device="cuda") * 0.05
    if c["fp8"]:
        sw = (w.abs().amax(1).clamp(min=1e-8) / 448.0).float()
        w = (w / sw[:, None]).to(E4M3)
    else:
        sw, w = None, w.to(BF16)
    bias = (torch.randn(N, generator=g, device="cuda") * 0.1).to(BF16) if c["bias"] else None
    res = padded(torch.randn(M, N, generator=g, device="cuda").to(BF16)) if c["res"] else None
    if ln is None:
        y = C.gemv_decode(x, w, sw, bias, res, c["act"])
    else:
        y = C.gemv_decode(x, w, sw, bias, res, c["act"], ln[0], ln[1], ln[2])
    ref, base = gemv_ref(x, w, sw, bias, c["act"], res, ln)
    key = f"gemv {'fp8' if c['fp8'] else 'bf16'}" + (f" ln {c['ln']}" if c["ln"] else f" K{K}")
    ck.bf16(key, f"gemv {cid}", y, ref, base)
    _report(ck)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the primitives (dispatch and activation ids), once each at a GPT / OPT shape
# ---------------------------------------------------------------------------------------------------------------------


@pytest.mark.gpu
def test_primitives_dispatch():
    from alpa_b200.ops import primitives as P
    ck = Checker()
    g = _gen(900, "cuda")
    T, H, F4 = 512, 1024, 4096                               # tokens, hidden, ffn of a small GPT
    x = torch.randn(4, T // 4, H, generator=g, device="cuda").to(BF16)
    w1 = (torch.randn(F4, H, generator=g, device="cuda") / H ** 0.5).to(BF16)
    b1 = torch.randn(F4, generator=g, device="cuda").to(BF16)
    xf, w1f = x.to(F64).reshape(T, H), w1.to(F64)
    for act, aid, did in (("gelu", ACT_GELU, ACT_DGELU), ("relu", ACT_RELU, ACT_DRELU)):
        y, z = P.linear_act(x, w1, b1, act)
        ref, base, zref, zbase, _ = epilogue_ref(xf @ w1f.t(), bias=b1, act=aid)
        ck.bf16(f"linear_act {act}", f"linear_act {act} y", y.reshape(T, F4), ref, base)
        ck.bf16(f"linear_act {act}", f"linear_act {act} z", z.reshape(T, F4), zref, zbase)
        # dgrad through w1: dz = (dy_h @ w1) * act'(z_h) with the activation input z of a [T, H] layer
        dyh = torch.randn(4, T // 4, F4, generator=g, device="cuda").to(BF16)
        zh = aux_in_values(T, H, g, "cuda").reshape(4, T // 4, H)
        dz = P.linear_dgrad_act(dyh, w1, zh, act)
        ref, base, _, _, _ = epilogue_ref(dyh.to(F64).reshape(T, F4) @ w1f, act=did, aux_in=zh.reshape(T, H))
        ck.bf16(f"linear_dgrad_act {act}", f"linear_dgrad_act {act}", dz.reshape(T, H), ref, base)
    # linear with bias, linear_dgrad, linear_wgrad
    y = P.linear(x, w1, b1)
    ref, base, _, _, _ = epilogue_ref(xf @ w1f.t(), bias=b1)
    ck.bf16("linear", "linear bias", y.reshape(T, F4), ref, base)
    dyh = torch.randn(4, T // 4, F4, generator=g, device="cuda").to(BF16)
    dx = P.linear_dgrad(dyh, w1)
    ref = dyh.to(F64).reshape(T, F4) @ w1f
    ck.bf16("linear_dgrad", "linear_dgrad", dx.reshape(T, H), ref, _bf(ref))
    dw = P.linear_wgrad(dyh, x)
    ref = dyh.to(F64).reshape(T, F4).t() @ xf
    ck.bf16("linear_wgrad", "linear_wgrad", dw, ref, _bf(ref))
    # layer_norm (output only; mean / rstd are checked with the kernel in tests/test_kernel_numerics.py)
    gam = (1 + 0.1 * torch.randn(H, generator=g, device="cuda")).to(BF16)
    bet = (0.1 * torch.randn(H, generator=g, device="cuda")).to(BF16)
    yn, _, _ = P.layer_norm(x, gam, bet, 1e-5)
    ref = ln_fwd_ref(x.reshape(T, H), gam, bet, 1e-5)[0]
    ck.bf16("layer_norm", "layer_norm", yn.reshape(T, H), ref, _bf(ref))
    # attention_qkvpacked (causal and full), baseline rounds the unnormalised P as the kernel does
    qkv = torch.randn(2, 256, 4, 3, 64, generator=g, device="cuda").to(BF16)
    for causal in (False, True):
        o, _ = P.attention_qkvpacked(qkv, 0.125, causal)
        q_, k_, v_ = (qkv[:, :, :, i] for i in range(3))
        vis = visible(256, 256, causal, device="cuda")
        ref, _ = attn_fwd_ref(q_, k_, v_, 0.125, vis)
        base, _ = attn_fwd_ref(q_, k_, v_, 0.125, vis, p_round=_bf)
        ck.bf16("attention_qkvpacked", f"attention_qkvpacked causal={causal}", o, ref, base)
    r = torch.randn(4, T // 4, H, generator=g, device="cuda").to(BF16)
    dx = P.linear_dgrad_add(dyh, w1, r)
    ref, base, _, _, _ = epilogue_ref(dyh.to(F64).reshape(T, F4) @ w1f, residual=r.reshape(T, H))
    ck.bf16("linear_dgrad_add", "linear_dgrad_add", dx.reshape(T, H), ref, base)
    bucket = Sentinel((F4, H), BF16)
    P._linear_wgrad_out(dyh, x, bucket.view)
    ref = dyh.to(F64).reshape(T, F4).t() @ xf
    ck.bf16("_linear_wgrad_out", "_linear_wgrad_out", bucket.view, ref, _bf(ref))
    ck.require(bucket.untouched_outside(), "_linear_wgrad_out wrote outside its bucket slice")
    # serving: OPT-2.7B projections
    xs = (torch.randn(96, 2560, generator=g, device="cuda") * 0.7).to(BF16)
    wq, sw = _fp8_w(2560, 2560, g)
    bs = (torch.randn(2560, generator=g, device="cuda") * 0.1).to(BF16)
    y = P.linear_fp8(xs, wq, sw, bs, "gelu")
    q, sx = _native().quantize_e4m3(xs)
    ref = act64((q.to(F64) @ wq.to(F64).t()) * sx.to(F64)[:, None] * sw.to(F64)[None, :] + bs.to(F64), ACT_GELU)
    ck.bf16("linear_fp8", "linear_fp8 gelu", y, ref, _bf(ref))
    wide = padded(xs, pad_cols=4)                             # row stride 2564: not a multiple of 8
    y2 = P.linear_fp8(wide, wq, sw, bs, "gelu")
    ck.require(torch.equal(y, y2), "linear_fp8 on a row stride that is not a multiple of 8 differs")
    wmx, wsf = (t.cuda() for t in P._quantize_mxfp8_ref(mx_operand(2560, 2560, g, "cuda").cpu()))
    y = P.linear_mxfp8(xs, wmx, wsf, bs, "relu")
    q, sf = _native().quantize_mxfp8(xs)
    ref = act64(mx_dequant64(q, sf) @ mx_dequant64(wmx, wsf).t() + bs.to(F64), ACT_RELU)
    ck.bf16("linear_mxfp8", "linear_mxfp8 relu", y, ref, _bf(ref))
    xd = torch.randn(1, 4, 2560, generator=g, device="cuda").to(BF16)
    rd = torch.randn(1, 4, 2560, generator=g, device="cuda").to(BF16)
    y = P.linear_decode(xd, wq, sw, bs, "relu", residual=rd)
    ref, base = gemv_ref(xd.reshape(4, 2560), wq, sw, bs, ACT_RELU, rd.reshape(4, 2560))
    ck.bf16("linear_decode", "linear_decode fp8 relu", y.reshape(4, 2560), ref, base)
    _report(ck)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: argument checks raise before any launch
# ---------------------------------------------------------------------------------------------------------------------


@pytest.mark.gpu
def test_bindings_reject_bad_views():
    C = _native()
    dev = "cuda"
    M, N, K = 64, 72, 64
    a = torch.randn(M, K, device=dev).to(BF16)
    b = torch.randn(N, K, device=dev).to(BF16)

    def flat_view(shape, dtype, offset, ld=None):
        ld = shape[-1] if ld is None else ld
        buf = torch.zeros(shape[0] * ld + offset + 16, device=dev, dtype=dtype)
        return buf[offset:offset + shape[0] * ld].view(shape[0], ld)[:, :shape[1]]

    def raises(fn, what):
        n0 = C.launch_count()
        with pytest.raises(RuntimeError):
            fn()
        torch.cuda.synchronize()
        assert C.launch_count() == n0, f"{what}: launched before raising"

    raises(lambda: C.gemm(a, b, out=flat_view((M, N), BF16, 0, ld=N + 1)), "gemm out with odd ldc")
    raises(lambda: C.gemm(a, b, out=flat_view((M, N), BF16, 1)), "gemm out 2-byte aligned")
    raises(lambda: C.gemm(a, b, out=flat_view((M, N), torch.float32, 1)), "gemm fp32 out 4-byte aligned")
    raises(lambda: C.gemm(a, b, aux_out=flat_view((M, N), BF16, 1), act=ACT_GELU), "gemm aux_out 2-byte aligned")
    raises(lambda: C.gemm(a, b, bias=torch.zeros(2 * N, device=dev, dtype=BF16)[::2]), "gemm strided bias")
    raises(lambda: C.gemm(a, b, bias=torch.zeros(N - 8, device=dev, dtype=BF16)), "gemm short bias")
    raises(lambda: C.gemm(a, b, bias=torch.zeros(N + 1, device=dev, dtype=BF16)[1:]), "gemm 2-byte aligned bias")
    raises(lambda: C.gemm(a, b, residual=torch.zeros(M, N, device=dev, dtype=BF16)[:M - 1]), "gemm short residual")
    raises(lambda: C.gemm(a, b, aux_in=torch.zeros(M, N, device=dev, dtype=BF16)[:, :N - 8].contiguous(),
                          act=ACT_DGELU), "gemm narrow aux_in")
    raises(lambda: C.gemm(a, b, aux_out=torch.zeros(M - 1, N, device=dev, dtype=BF16), act=ACT_GELU),
           "gemm short aux_out")
    raises(lambda: C.gemm(a.repeat(3, 1, 1), b.repeat(3, 1, 1), out=torch.zeros(2, M, N, device=dev, dtype=BF16)),
           "gemm out with fewer batches than the operands")
    wq = torch.zeros(N, K, device=dev).to(E4M3)
    sw = torch.ones(N, device=dev)
    x_ld = torch.zeros(M, K + 4, device=dev, dtype=BF16)[:, :K]             # row stride 68
    x_off = torch.zeros(M, K + 8, device=dev, dtype=BF16)[:, 4:4 + K]       # base 8 bytes past a 16-byte boundary
    for x, what in ((x_ld, "row stride 68"), (x_off, "8-byte aligned base")):
        raises(lambda: C.gemm_fp8(x, wq, sw, None, 0), f"gemm_fp8 x {what}")
        raises(lambda: C.quantize_e4m3(x), f"quantize_e4m3 x {what}")
        raises(lambda: C.quantize_mxfp8(x), f"quantize_mxfp8 x {what}")
    raises(lambda: C.gemm_fp8(a, wq, sw, torch.zeros(N, device=dev), 0), "gemm_fp8 fp32 bias")
    raises(lambda: C.gemm_fp8(a, wq, sw, torch.zeros(N - 8, device=dev, dtype=BF16), 0), "gemm_fp8 short bias")
    raises(lambda: C.gemv_decode(x_off[:4], b), "gemv_decode x 8-byte aligned base")
