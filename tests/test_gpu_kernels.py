"""Numerics of the sm_90a kernels against fp32 PyTorch references (run with -m gpu on an H100)."""
import importlib

import pytest
import torch

pytestmark = pytest.mark.gpu


def _run(section):
    gc = importlib.import_module("scripts.gpu_check")
    gc.FAILS.clear()
    getattr(gc, section)()
    assert not gc.FAILS, gc.FAILS


def test_native_extension_loaded():
    from alpa_b200 import ops
    assert ops.native_available(), "sm_90a extension must be built in-tree (python -m alpa_b200.ops.build)"
    assert hasattr(ops.native_module(), "gemm")


def test_gemm_numerics():
    _run("sec_gemm")


def test_layernorm_ce_embedding_adam_numerics():
    _run("sec_misc")


def test_moe_kernels_numerics():
    _run("sec_moe")


def test_fp8_gemm_numerics():
    _run("sec_fp8")


def test_decode_gemv_numerics():
    _run("sec_gemv")


def test_attention_numerics():
    gc = importlib.import_module("scripts.gpu_check")
    from scripts import gpu_check_attn
    gc.FAILS.clear()
    gpu_check_attn.run(gc.check, gc.timeit, gc.FAILS)
    assert not gc.FAILS, gc.FAILS


def test_primitives_match_reference_on_gpu():
    """Every primitive: native bf16 result vs the fp32 PyTorch implementation of the same op."""
    from alpa_b200 import ops
    torch.manual_seed(0)
    dev = "cuda"
    x = torch.randn(4, 128, 256, device=dev, dtype=torch.bfloat16)
    w = torch.randn(512, 256, device=dev, dtype=torch.bfloat16) * 0.05
    b = torch.randn(512, device=dev, dtype=torch.bfloat16)
    y = ops.linear(x, w, b)
    ref = torch.nn.functional.linear(x.float(), w.float(), b.float())
    assert (y.float() - ref).abs().max() < 0.1
    h, z = ops.linear_act(x, w, b, "gelu")
    assert (h.float() - torch.nn.functional.gelu(ref)).abs().max() < 0.1
    dy = torch.randn_like(y)
    dx = ops.linear_dgrad(dy, w)
    assert (dx.float() - dy.float() @ w.float()).abs().max() < 0.3
    dw = ops.linear_wgrad(dy, x)
    assert (dw.float() - dy.float().reshape(-1, 512).t() @ x.float().reshape(-1, 256)).abs().max() < 1.5
    dz = ops.primitives.linear_dgrad_act(torch.randn(4, 128, 256, device=dev, dtype=torch.bfloat16),
                                         torch.randn(256, 512, device=dev, dtype=torch.bfloat16) * 0.05, z, "gelu")
    assert torch.isfinite(dz.float()).all()
    g = torch.ones(256, device=dev, dtype=torch.bfloat16)
    be = torch.zeros(256, device=dev, dtype=torch.bfloat16)
    yn, mean, rstd = ops.layer_norm(x, g, be, 1e-5)
    assert (yn.float() - torch.nn.functional.layer_norm(x.float(), (256,))).abs().max() < 0.05
    qkv = torch.randn(2, 256, 4, 3, 64, device=dev, dtype=torch.bfloat16)
    o, lse = ops.attention_qkvpacked(qkv, 0.125, False)
    q, k, v = (qkv[:, :, :, i].float().permute(0, 2, 1, 3) for i in range(3))
    ref_o = torch.softmax(q @ k.transpose(-1, -2) * 0.125, -1) @ v
    assert (o.float() - ref_o.permute(0, 2, 1, 3)).abs().max() < 0.05


def test_train_step_decreases_loss():
    import __graft_entry__ as g
    g.smoke()
