"""RMSNorm, rotary embedding and SwiGLU kernels against float64 references, and the bf16 Llama-style model on the GPU.

The rules are those of tests/test_kernel_numerics.py: bf16 outputs within RATIO = 2 of a baseline that computes in
float64 from the same bf16 inputs and rounds only the output (each kernel rounds once), fp32 outputs (rstd, dgamma)
within TOL32 * sum |terms|.  The rotary reference takes float64 cos / sin of the same fp32 angle float(pos) * inv_freq
that the kernel and HF form.  Whole-model checks compare the kernels' bf16 result and the PyTorch path's bf16 result with
an fp32 (or float64) reference under the same bf16 rule.
"""
import copy
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernel_numerics import BF16, F64, LN_H, Checker, _bf, _ln_rows, _report  # noqa: E402

from alpa_b200.global_env import global_config  # noqa: E402
from alpa_b200.ops import primitives as P  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _own_fallback_record(monkeypatch):
    """Each test sees only the library fallbacks it records itself."""
    monkeypatch.setattr(P, "_FALLBACK_SEEN", set())


def _native():
    from alpa_b200 import ops
    return ops.native_module()


# ---- RMSNorm: every LayerNorm size, both kernel families, both grid regimes ----------------------------------------
def _rms_cases():
    sms = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
    return [(H, rows, res) for H in LN_H for rows in _ln_rows(H, sms) for res in (False, True)]


@pytest.mark.parametrize("H,rows,res", _rms_cases())
def test_rms_norm(H, rows, res):
    C = _native()
    gen = torch.Generator(device="cuda").manual_seed(H * 5 + rows)
    x = (2 + torch.randn(rows, H, device="cuda", generator=gen)).to(BF16)
    r = torch.randn(rows, H, device="cuda", generator=gen).to(BF16) if res else None
    g = (1 + 0.5 * torch.randn(H, device="cuda", generator=gen)).to(BF16)
    dy = torch.randn(rows, H, device="cuda", generator=gen).to(BF16)
    name = f"rms H={H} rows={rows}{' +res' if res else ''}"
    ck = Checker()
    outs = [C.layernorm_fwd(x, r, g, None, 1e-5, res, rms=True) for _ in range(2)]
    y, mean, rstd, s = outs[0]
    ck.require(mean is None, f"{name}: RMSNorm returned a mean")
    ck.require(all(torch.equal(a, b) for a, b in zip(outs[0][::2], outs[1][::2]) if a is not None),
               f"{name}: forward differs between two runs")
    if res:
        s_ref = x.to(F64) + r.to(F64)
        ck.bf16("rmsnorm fwd sum_out", f"{name} sum_out", s, s_ref, _bf(s_ref))
        xin = (x.float() + r.float()).to(BF16)               # the kernel normalises the bf16 sum it stores
    else:
        xin = x
    xf = xin.to(F64)
    ms = xf.pow(2).mean(-1)
    r_ref = (ms + 1e-5).rsqrt()
    y_ref = xf * r_ref[:, None] * g.to(F64)
    ck.bf16("rmsnorm fwd y", f"{name} y", y, y_ref, _bf(y_ref))
    ck.fp32("rmsnorm fwd rstd", f"{name} rstd", rstd, r_ref, r_ref * ms / (ms + 1e-5))
    # the backward's reference starts from the forward's fp32 rstd (checked above)
    rs = rstd.to(F64)
    xh = xf * rs[:, None]
    gd = dy.to(F64) * g.to(F64)
    dx_ref = rs[:, None] * (gd - xh * (gd * xh).mean(-1, keepdim=True))
    dg_ref, t_dg = (dy.to(F64) * xh).sum(0), (dy.to(F64) * xh).abs().sum(0)
    bwd = []
    for _ in range(2):
        dg = torch.zeros(H, device="cuda")
        bwd.append((C.layernorm_bwd(dy, xin, g, None, rstd, r, dg, None, rms=True), dg))
    dx, dg = bwd[0]
    want = dx_ref + (r.to(F64) if res else 0.0)
    ck.bf16("rmsnorm bwd dx" + (" + dres" if res else ""), f"{name} dx", dx, want, _bf(want))
    ck.fp32("rmsnorm bwd dgamma", f"{name} dgamma", dg, dg_ref, t_dg)
    ck.require(torch.equal(bwd[0][0], bwd[1][0]) and torch.equal(bwd[0][1], bwd[1][1]),
               f"{name}: dx / dgamma differ between two runs")
    _report(ck)


# ---- rotary --------------------------------------------------------------------------------------------------------
def _positions(B, S, kind, gen):
    if kind == "far":
        return torch.randint(0, 65536, (B, S), device="cuda", generator=gen)
    # packed sequences: positions restart mid-row
    pos = torch.arange(S, device="cuda").repeat(B, 1)
    cut = S // 3
    pos[:, cut:] -= cut
    pos[1:, 2 * cut:] = torch.arange(S - 2 * cut, device="cuda") + 60000
    return pos


@pytest.mark.parametrize("G", [1, 4, 8])
@pytest.mark.parametrize("Hkv", [1, 8])
@pytest.mark.parametrize("D", [64, 80, 96, 128])
@pytest.mark.parametrize("kind", ["far", "packed"])
def test_rotary(G, Hkv, D, kind):
    gen = torch.Generator(device="cuda").manual_seed(G * 100 + Hkv * 10 + D)
    B, S, theta = 2, 77, 500000.0
    qkv = torch.randn(B, S, Hkv, G + 2, D, device="cuda", generator=gen).to(BF16)
    pos = _positions(B, S, kind, gen)
    inv = P._inv_freq(D, theta, "cuda:0")
    ang = (pos.float()[..., None] * inv).to(F64)                   # the fp32 angle, then float64 cos / sin
    c, s = ang.cos()[:, :, None, None], ang.sin()[:, :, None, None]
    x = qkv[:, :, :, :G + 1].to(F64)
    x1, x2 = x[..., :D // 2], x[..., D // 2:]
    ck = Checker()
    name = f"rotary G={G} Hkv={Hkv} D={D} {kind}"
    for inverse in (False, True):
        sg = -s if inverse else s
        ref = torch.cat([x1 * c - x2 * sg, x2 * c + x1 * sg], -1)
        out = P.rotary_packed(qkv, pos, theta, inverse)
        ck.bf16("rotary" + (" inverse" if inverse else ""), f"{name} inverse={inverse}", out[:, :, :, :G + 1], ref,
                _bf(ref))
        ck.require(torch.equal(out[:, :, :, G + 1], qkv[:, :, :, G + 1]), f"{name}: V not copied bitwise")
    assert P.library_fallbacks() == [], P.library_fallbacks()
    _report(ck)


def test_rotary_position_ids_forms():
    """The kernel takes [1, S] and int32 positions like the reference, and refuses positions on another device."""
    gen = torch.Generator(device="cuda").manual_seed(5)
    qkv = torch.randn(3, 64, 2, 6, 64, device="cuda", generator=gen).to(BF16)
    pos = torch.arange(64, device="cuda") + 1000
    want = P.rotary_packed(qkv, pos.repeat(3, 1), 10000.0, False)
    assert torch.equal(P.rotary_packed(qkv, pos[None], 10000.0, False), want)
    assert torch.equal(P.rotary_packed(qkv, pos.repeat(3, 1).to(torch.int32), 10000.0, False), want)
    assert P.library_fallbacks() == [], P.library_fallbacks()
    with pytest.raises(RuntimeError):
        P.rotary_packed(qkv, pos.repeat(3, 1).cpu(), 10000.0, False)
    with pytest.raises(RuntimeError, match="one CUDA device"):
        _native().rotary_packed(qkv, pos.repeat(3, 1).cpu(), P._inv_freq(64, 10000.0, "cuda:0"), False)


# ---- SwiGLU --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,I", [(1, 4), (7, 12), (4096, 1376), (16384, 5504)])
def test_swiglu(rows, I):
    gen = torch.Generator(device="cuda").manual_seed(rows + I)
    g = torch.randn(rows * I, device="cuda", generator=gen) * 3
    far = g[::17]
    g[::17] = 80 * (torch.rand(far.numel(), device="cuda", generator=gen) * 2 - 1)   # some gates out to |g| ~ 80
    gu = torch.stack([g.view(rows, I), torch.randn(rows, I, device="cuda", generator=gen)], -1).to(BF16)
    dh = torch.randn(rows, I, device="cuda", generator=gen).to(BF16)
    g, u = gu[..., 0].to(F64), gu[..., 1].to(F64)
    sg = torch.sigmoid(g)
    h_ref = g * sg * u
    dg_ref = dh.to(F64) * u * sg * (1 + g * (1 - sg))
    du_ref = dh.to(F64) * g * sg
    h = P.swiglu(gu)
    dgu = P.swiglu_bwd(dh, gu)
    name = f"swiglu rows={rows} I={I}"
    ck = Checker()
    ck.bf16("swiglu fwd", f"{name} h", h, h_ref, _bf(h_ref))
    ck.bf16("swiglu bwd dg", f"{name} dg", dgu[..., 0], dg_ref, _bf(dg_ref))
    ck.bf16("swiglu bwd du", f"{name} du", dgu[..., 1], du_ref, _bf(du_ref))
    assert P.library_fallbacks() == [], P.library_fallbacks()
    _report(ck)


# ---- kernel or reference ------------------------------------------------------------------------------------------
def _rn(*shape):
    return torch.randn(*shape, generator=torch.Generator(device="cuda").manual_seed(0), device="cuda").to(BF16)


def _calls(H, D, I):
    pos = torch.arange(32, device="cuda").repeat(2, 1)
    x, r, g = _rn(16, H), _rn(16, H), _rn(H)
    rstd = x.float().pow(2).mean(-1).add(1e-5).rsqrt()
    return {"rms_norm": lambda: P.rms_norm(x, g, 1e-5), "add_rms_norm": lambda: P.add_rms_norm(x, r, g, 1e-5),
            "rms_norm_bwd": lambda: P.rms_norm_bwd(r, x, g, rstd, None),
            "rotary_packed": lambda: P.rotary_packed(_rn(2, 32, 2, 4, D), pos, 10000.0, False),
            "swiglu": lambda: P.swiglu(_rn(2, 32, I, 2)), "swiglu_bwd": lambda: P.swiglu_bwd(_rn(2, 32, I), _rn(2, 32, I, 2))}


@pytest.mark.parametrize("op", ["rms_norm", "add_rms_norm", "rms_norm_bwd", "rotary_packed", "swiglu", "swiglu_bwd"])
def test_kernel_or_recorded_fallback(op):
    C = _native()
    n0 = C.launch_count()
    _calls(256, 64, 64)[op]()
    torch.cuda.synchronize()
    assert C.launch_count() > n0 and P.library_fallbacks() == [], (op, P.library_fallbacks())
    got = _calls(8200, 72, 6)[op]()                # H > 8192, D % 16 != 0, I % 4 != 0
    rec = P.library_fallbacks()
    assert len(rec) == 1 and rec[0][0] == op, rec
    global_config.use_native_kernels = False
    try:
        want = _calls(8200, 72, 6)[op]()
    finally:
        global_config.use_native_kernels = True
    for a, b in zip(got if isinstance(got, tuple) else (got,), want if isinstance(want, tuple) else (want,)):
        assert torch.equal(a, b), op


# ---- whole model ---------------------------------------------------------------------------------------------------
def _llama_run(model, params, ids, pos, labels):
    from alpa_b200.model.gpt_model import gpt_lm_loss
    from alpa_b200.model.model_util import functional_call
    params = {k: v.detach().clone().requires_grad_() for k, v in params.items()}
    logits = functional_call(model, params, (ids, pos))
    grads = torch.autograd.grad(gpt_lm_loss(logits, labels), list(params.values()))
    return logits.detach(), dict(zip(params, grads))


def test_llama_model_kernels_against_reference_path():
    """bf16 GPTModel(arch="llama") with the kernels and with the PyTorch path, both against the fp32 model."""
    from alpa_b200.model.gpt_model import GPTConfig, GPTModel
    from alpa_b200.model.model_util import params_of
    cfg = GPTConfig(arch="llama", vocab_size=1024, hidden_size=256, num_hidden_layers=2, num_attention_heads=8,
                    num_key_value_heads=2, intermediate_size=512, causal=True, dtype=BF16)
    torch.manual_seed(0)
    model = GPTModel(cfg, device="cuda")
    params = params_of(model)
    B, S = 2, 128
    ids = torch.randint(1, 1024, (B, S), device="cuda")
    pos = torch.arange(S, device="cuda").repeat(B, 1) + torch.tensor([[0], [1000]], device="cuda")
    labels = torch.randint(1, 1024, (B, S), device="cuda")
    n0 = _native().launch_count()
    k_logits, k_grads = _llama_run(model, params, ids, pos, labels)
    assert _native().launch_count() > n0 and P.library_fallbacks() == [], P.library_fallbacks()
    global_config.use_native_kernels = False
    try:
        r_logits, r_grads = _llama_run(model, params, ids, pos, labels)
        model32 = GPTModel(GPTConfig(**{**cfg.__dict__, "dtype": torch.float32}), device="cuda")
        f_logits, f_grads = _llama_run(model32, {k: v.float() for k, v in params.items()}, ids, pos, labels)
    finally:
        global_config.use_native_kernels = True
    ck = Checker()
    ck.bf16("llama model logits", "logits", k_logits, f_logits, r_logits)
    for k in params:
        ck.bf16("llama model grads", f"grad {k}", k_grads[k], f_grads[k], r_grads[k])
    _report(ck)


@pytest.mark.parametrize("offset", [0, 30000])
def test_hf_llama_parity_bf16(offset):
    """The converted bf16 model's logits are no further from HF's float64 logits than 2x HF's own bf16 logits are."""
    transformers = pytest.importorskip("transformers")
    from alpa_b200.model.gpt_model import GPTModel, llama_config_from_hf, llama_params_from_hf
    from alpa_b200.model.model_util import functional_call
    torch.manual_seed(0)
    hcfg = transformers.LlamaConfig(vocab_size=512, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                                    num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=65536,
                                    rms_norm_eps=1e-5, attn_implementation="eager")
    hf = transformers.LlamaForCausalLM(hcfg).eval()
    cfg = llama_config_from_hf(hcfg, dtype=BF16)
    model = GPTModel(cfg, device="cuda")
    params = {k: v.cuda() for k, v in llama_params_from_hf(hf.state_dict(), cfg).items()}
    B, S = 2, 64
    ids = torch.randint(0, 512, (B, S), device="cuda")
    pos = torch.arange(S, device="cuda").repeat(B, 1) + offset
    hf_bf16 = copy.deepcopy(hf).to(device="cuda", dtype=BF16)
    hf_bf16.model.rotary_emb.inv_freq = hf.model.rotary_emb.inv_freq.cuda()    # HF keeps its frequencies in fp32
    with torch.no_grad():
        ours = functional_call(model, params, (ids, pos)).to(F64)
        hb = hf_bf16(input_ids=ids, position_ids=pos).logits.to(F64)
        f64 = hf.to(device="cuda", dtype=F64)(input_ids=ids, position_ids=pos).logits
    e_ours, e_hf = (ours - f64).norm().item(), (hb - f64).norm().item()
    assert e_ours <= 2 * e_hf, f"offset {offset}: |ours - f64| {e_ours:.4e} > 2 x |hf bf16 - f64| {e_hf:.4e}"
    assert P.library_fallbacks() == [], P.library_fallbacks()
