"""Primitive operators (torch.library custom ops, namespace ``alpa_b200``).

See ``alpa_b200/ops/__init__.py`` for the contract.  The reference has no counterpart file: its
primitives are XLA HLO ops lowered to cuBLAS / LLVM fusions (SURVEY.md §2.5 K1-K9); here they are the
hand-written sm_90a kernels, and the *same* op names appear in traced graphs, plans and programs.
"""
from __future__ import annotations

import math
from functools import cache
from typing import List, NamedTuple, Optional, Tuple, Union

import torch
import torch.nn.functional as F
from torch import Tensor

from alpa_b200.global_env import global_config

__all__ = [
    "linear", "linear_act", "linear_dgrad", "linear_dgrad_add", "linear_wgrad", "bias_grad", "act_bwd", "layer_norm",
    "add_layer_norm", "layer_norm_bwd", "rms_norm", "add_rms_norm", "rms_norm_bwd", "rotary_packed", "swiglu",
    "swiglu_bwd", "attention", "attention_bwd", "attention_gqa_packed",
    "attention_gqa_packed_bwd", "embedding", "embedding_bwd",
    "cross_entropy", "cross_entropy_bwd", "fused_adamw_", "pipeline_marker",
    "bmm", "moe_dispatch", "moe_combine", "moe_combine_wgrad", "moe_top2_route", "linear_fp8", "linear_decode", "RMSNormArgs", "decode_attention", "decode_attention_gqa", "ragged_attention",
    "paged_prefill_attention", "lora_shrink", "lora_expand_",
    "Fp8KV", "kv_cache_store", "kv_cache_load", "kv_cache_nbytes",
    "attention_cached", "attention_cached_", "quantize_mxfp8", "dequantize_mxfp8", "linear_mxfp8", "mx_pack_scale_atoms",
    "mx_unpack_scale_atoms", "pack_tiles", "unpack_tiles", "packed_nbytes",
    "dropout", "dropout_like", "dropout_keep_mask",
]

_ACT_IDS = {"none": 0, "gelu": 1, "relu": 2}
_DACT_IDS = {"gelu": 3, "relu": 4}


_FALLBACK_SEEN = set()


def _kernels(op: str, *tensors: Optional[Tensor], dtypes=(torch.bfloat16,), unsupported=None):
    """The sm_90a extension if its kernel serves this call of `op`, else None (the caller runs its PyTorch reference).

    Expected reference paths return None silently: a tensor off CUDA, `global_config.use_native_kernels` off, or a
    floating tensor whose dtype is not in `dtypes` (None: any dtype).  A missing extension is an error unless
    ALPA_B200_ALLOW_FALLBACK=1.  `unsupported` is the caller's reason why the kernel cannot take this layout, or a
    function returning it (called only past the checks above, so the reference path builds no kernel operand views);
    such a call is a library fallback: it is recorded for `library_fallbacks()`, warned about once, and returns None."""
    ts = [t for t in tensors if t is not None]
    if not ts or not global_config.use_native_kernels or not all(t.is_cuda for t in ts):
        return None
    if dtypes is not None and not all(t.dtype in dtypes for t in ts if t.is_floating_point()):
        return None
    from alpa_b200 import ops
    if not ops.native_available():
        if ops.allow_fallback():
            return None
        raise RuntimeError(f"alpa_b200: {op} on CUDA but the sm_90a extension is not built/loaded "
                           "(run `python -m alpa_b200.ops.build`; set ALPA_B200_ALLOW_FALLBACK=1 to use PyTorch)")
    if callable(unsupported):
        unsupported = unsupported()
    if unsupported is not None:
        key = (op, unsupported, tuple((tuple(t.shape), tuple(t.stride())) for t in ts))
        if key not in _FALLBACK_SEEN:
            _FALLBACK_SEEN.add(key)
            import logging
            logging.getLogger(__name__).warning(
                "alpa_b200: %s falls back to PyTorch (%s; operand shapes / strides %s)", *key)
        return None
    return ops.native_module()


def library_fallbacks():
    """(op, reason, operand shapes / strides) of every call that ran a PyTorch reference on CUDA although the sm_90a
    extension is loaded, because the kernel cannot take the operands' layout.  One warning per distinct entry is
    logged; tests and benchmarks can assert this stays empty."""
    return sorted(_FALLBACK_SEEN)


def _gemm_unsupported(*mats: Tensor) -> Optional[str]:
    """Why the wgmma GEMM's TMA descriptors cannot describe these operands, or None."""
    for m in mats:
        if m.dim() not in (2, 3) or m.stride(-1) != 1 or m.shape[-1] % 8 or m.shape[-2] % 8:
            return "GEMM operand shape"
        if m.stride(-2) % 8 or m.data_ptr() % 16:
            return "GEMM operand alignment"
    return None


def _as2d(x: Tensor) -> Tensor:
    x2 = x.reshape(-1, x.shape[-1])
    return x2 if x2.stride(-1) == 1 else x2.contiguous()


def _act_fn(z: Tensor, act: str) -> Tensor:
    if act == "gelu":
        return F.gelu(z)
    if act == "relu":
        return F.relu(z)
    if act == "none":
        return z
    raise ValueError(act)


# =================================================================================================
# linear family
# =================================================================================================
@torch.library.custom_op("alpa_b200::linear", mutates_args=())
def linear(x: Tensor, w: Tensor, b: Optional[Tensor] = None) -> Tensor:
    """y[..., N] = x[..., K] @ w[N, K]^T + b[N]"""
    x2 = cache(lambda: _as2d(x))
    if C := _kernels("linear", x, w, b, unsupported=lambda: _gemm_unsupported(x2(), w)):
        return C.gemm(x2(), w, False, False, bias=b).view(*x.shape[:-1], w.shape[0])
    return F.linear(x, w, b)


@linear.register_fake
def _(x, w, b=None):
    return x.new_empty(*x.shape[:-1], w.shape[0])


@torch.library.custom_op("alpa_b200::linear_act", mutates_args=())
def linear_act(x: Tensor, w: Tensor, b: Optional[Tensor], act: str) -> Tuple[Tensor, Tensor]:
    """(act(z), z) with z = x @ w^T + b; the pre-activation z is kept for the backward pass."""
    x2 = cache(lambda: _as2d(x))
    if C := _kernels("linear_act", x, w, b, unsupported=lambda: _gemm_unsupported(x2(), w)):
        z = torch.empty(x2().shape[0], w.shape[0], device=x.device, dtype=x.dtype)
        y = C.gemm(x2(), w, False, False, bias=b, aux_out=z, act=_ACT_IDS[act])
        shp = (*x.shape[:-1], w.shape[0])
        return y.view(shp), z.view(shp)
    z = F.linear(x, w, b)
    return _act_fn(z, act), z


@linear_act.register_fake
def _(x, w, b, act):
    y = x.new_empty(*x.shape[:-1], w.shape[0])
    return y, torch.empty_like(y)


@torch.library.custom_op("alpa_b200::linear_dgrad", mutates_args=())
def linear_dgrad(dy: Tensor, w: Tensor) -> Tensor:
    """dx[..., K] = dy[..., N] @ w[N, K]"""
    d2 = cache(lambda: _as2d(dy))
    if C := _kernels("linear_dgrad", dy, w, unsupported=lambda: _gemm_unsupported(d2(), w)):
        return C.gemm(d2(), w, False, True).view(*dy.shape[:-1], w.shape[1])
    return torch.matmul(dy, w)


@linear_dgrad.register_fake
def _(dy, w):
    return dy.new_empty(*dy.shape[:-1], w.shape[1])


@torch.library.custom_op("alpa_b200::linear_dgrad_act", mutates_args=())
def linear_dgrad_act(dy: Tensor, w: Tensor, z: Tensor, act: str) -> Tensor:
    """dz = (dy @ w) * act'(z): the activation backward fused into the dgrad epilogue."""
    v = cache(lambda: (_as2d(dy), _as2d(z)))
    if C := _kernels("linear_dgrad_act", dy, w, z, unsupported=lambda: _gemm_unsupported(v()[0], w) or (
                     None if v()[1].is_contiguous() else "pre-activation not contiguous")):
        d2, z2 = v()
        return C.gemm(d2, w, False, True, aux_in=z2, act=_DACT_IDS[act]).view(*dy.shape[:-1], w.shape[1])
    return _act_bwd_ref(torch.matmul(dy, w), z, act)


@linear_dgrad_act.register_fake
def _(dy, w, z, act):
    return dy.new_empty(*dy.shape[:-1], w.shape[1])


@torch.library.custom_op("alpa_b200::linear_dgrad_add", mutates_args=())
def linear_dgrad_add(dy: Tensor, w: Tensor, r: Optional[Tensor]) -> Tensor:
    """dx = dy @ w + r: the accumulation of a second gradient contribution (residual branch) fused into the dgrad
    GEMM epilogue (one read of r instead of a separate read-read-write add kernel).  `r` is None on the devices of a
    tensor-parallel group that must not add it again (dx is a partial sum there)."""
    if r is None:
        return linear_dgrad._init_fn(dy, w)
    v = cache(lambda: (_as2d(dy), _as2d(r)))
    if C := _kernels("linear_dgrad_add", dy, w, r, unsupported=lambda: _gemm_unsupported(v()[0], w) or (
                     None if v()[1].is_contiguous() and v()[1].shape == (v()[0].shape[0], w.shape[1])
                     else "addend not a contiguous [M, K]")):
        d2, r2 = v()
        return C.gemm(d2, w, False, True, residual=r2).view(*dy.shape[:-1], w.shape[1])
    return torch.matmul(dy, w) + r


@linear_dgrad_add.register_fake
def _(dy, w, r):
    return dy.new_empty(*dy.shape[:-1], w.shape[1])


@torch.library.custom_op("alpa_b200::linear_wgrad", mutates_args=())
def linear_wgrad(dy: Tensor, x: Tensor) -> Tensor:
    """dw[N, K] = dy[..., N]^T @ x[..., K]"""
    v = cache(lambda: (_as2d(dy), _as2d(x)))
    if C := _kernels("linear_wgrad", dy, x, unsupported=lambda: _gemm_unsupported(*v())):
        return C.gemm(*v(), True, True)
    d2 = dy.reshape(-1, dy.shape[-1])
    x2 = x.reshape(-1, x.shape[-1])
    return torch.matmul(d2.t(), x2)


@linear_wgrad.register_fake
def _(dy, x):
    return dy.new_empty(dy.shape[-1], x.shape[-1])


@torch.library.custom_op("alpa_b200::bias_grad", mutates_args=())
def bias_grad(dy: Tensor) -> Tensor:
    """db[N] = sum over all leading dims of dy[..., N]"""
    d2 = cache(lambda: _as2d(dy))
    if C := _kernels("bias_grad", dy, unsupported=lambda: None if d2().shape[1] % 8 == 0 and d2().stride(0) % 8 == 0
                     and d2().data_ptr() % 16 == 0 else "rows not 16-byte aligned"):
        out = torch.zeros(dy.shape[-1], device=dy.device, dtype=torch.float32)
        C.colsum_(d2(), out)
        return out.to(dy.dtype)
    return dy.reshape(-1, dy.shape[-1]).sum(0)


@bias_grad.register_fake
def _(dy):
    return dy.new_empty(dy.shape[-1])


def _act_bwd_ref(dy: Tensor, z: Tensor, act: str) -> Tensor:
    if act == "gelu":
        zf = z.float()
        cdf = 0.5 * (1.0 + torch.erf(zf * 0.7071067811865476))
        pdf = torch.exp(-0.5 * zf * zf) * 0.3989422804014327
        return (dy.float() * (cdf + zf * pdf)).to(dy.dtype)
    if act == "relu":
        return torch.where(z > 0, dy, torch.zeros_like(dy))
    if act == "none":
        return dy
    raise ValueError(act)


@torch.library.custom_op("alpa_b200::act_bwd", mutates_args=())
def act_bwd(dy: Tensor, z: Tensor, act: str) -> Tensor:
    """dz = dy * act'(z)"""
    return _act_bwd_ref(dy, z, act)


@act_bwd.register_fake
def _(dy, z, act):
    return torch.empty_like(dy)


def _linear_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)  # unused outputs yield None, not a zero tensor + add
    x, w, b = inputs
    ctx.save_for_backward(x, w)
    ctx.has_bias = b is not None


def _linear_bwd(ctx, dy):
    if dy is None:
        return None, None, None
    x, w = ctx.saved_tensors
    dx = linear_dgrad(dy, w) if ctx.needs_input_grad[0] else None
    dw = linear_wgrad(dy, x) if ctx.needs_input_grad[1] else None
    db = bias_grad(dy) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
    return dx, dw, db


linear.register_autograd(_linear_bwd, setup_context=_linear_setup)


def _linear_act_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)  # unused outputs yield None, not a zero tensor + add
    x, w, b, act = inputs
    _, z = output
    ctx.save_for_backward(x, w, z)
    ctx.has_bias = b is not None
    ctx.act = act


def _linear_act_bwd(ctx, dy, dz_extra):
    x, w, z = ctx.saved_tensors
    if dy is None and dz_extra is None:
        return None, None, None, None
    dz = act_bwd(dy, z, ctx.act) if dy is not None else None
    if dz_extra is not None:
        dz = dz_extra if dz is None else dz + dz_extra
    dx = linear_dgrad(dz, w) if ctx.needs_input_grad[0] else None
    dw = linear_wgrad(dz, x) if ctx.needs_input_grad[1] else None
    db = bias_grad(dz) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
    return dx, dw, db, None


linear_act.register_autograd(_linear_act_bwd, setup_context=_linear_act_setup)


# =================================================================================================
# layer norm
# =================================================================================================
def _ln_ref(x: Tensor, g: Tensor, b: Tensor, eps: float):
    xf = x.float()
    mean = xf.mean(-1)
    var = xf.var(-1, unbiased=False)
    rstd = torch.rsqrt(var + eps)
    y = (xf - mean[..., None]) * rstd[..., None] * g.float() + b.float()
    return y.to(x.dtype), mean, rstd


def _ln_unsupported(H: int) -> Optional[str]:
    """Why the LayerNorm kernels (8-element vectors, at most 8192 elements per row) cannot take rows of H, or None."""
    return None if H % 8 == 0 and H <= 8192 else "row length not a multiple of 8 up to 8192"


@torch.library.custom_op("alpa_b200::layer_norm", mutates_args=())
def layer_norm(x: Tensor, g: Tensor, b: Tensor, eps: float) -> Tuple[Tensor, Tensor, Tensor]:
    """(y, mean, rstd); statistics are fp32 with shape x.shape[:-1]."""
    if C := _kernels("layer_norm", x, g, b, unsupported=_ln_unsupported(x.shape[-1])):
        y, mean, rstd, _ = C.layernorm_fwd(x.contiguous(), None, g, b, eps, False)
        return y, mean.view(x.shape[:-1]), rstd.view(x.shape[:-1])
    return _ln_ref(x, g, b, eps)


@layer_norm.register_fake
def _(x, g, b, eps):
    st = x.new_empty(x.shape[:-1], dtype=torch.float32)
    return torch.empty_like(x), st, torch.empty_like(st)


@torch.library.custom_op("alpa_b200::add_layer_norm", mutates_args=())
def add_layer_norm(x: Tensor, r: Tensor, g: Tensor, b: Tensor, eps: float) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """s = x + r; (layer_norm(s), s, mean, rstd) in one pass."""
    if C := _kernels("add_layer_norm", x, r, g, b, unsupported=_ln_unsupported(x.shape[-1])):
        y, mean, rstd, s = C.layernorm_fwd(x.contiguous(), r.contiguous(), g, b, eps, True)
        return y, s, mean.view(x.shape[:-1]), rstd.view(x.shape[:-1])
    s = x + r
    y, mean, rstd = _ln_ref(s, g, b, eps)
    return y, s, mean, rstd


@add_layer_norm.register_fake
def _(x, r, g, b, eps):
    st = x.new_empty(x.shape[:-1], dtype=torch.float32)
    return torch.empty_like(x), torch.empty_like(x), st, torch.empty_like(st)


@torch.library.custom_op("alpa_b200::layer_norm_bwd", mutates_args=())
def layer_norm_bwd(dy: Tensor, x: Tensor, g: Tensor, mean: Tensor, rstd: Tensor,
                   dres: Optional[Tensor]) -> Tuple[Tensor, Tensor, Tensor]:
    """(dx [+ dres], dgamma, dbeta) of y = layer_norm(x)."""
    H = x.shape[-1]
    if C := _kernels("layer_norm_bwd", dy, x, g, unsupported=_ln_unsupported(H)):
        dg = torch.zeros(H, device=x.device, dtype=torch.float32)
        db = torch.zeros(H, device=x.device, dtype=torch.float32)
        dx = C.layernorm_bwd(dy.contiguous(), x.contiguous(), g, mean.reshape(-1).contiguous(),
                             rstd.reshape(-1).contiguous(), dres.contiguous() if dres is not None else None, dg, db)
        return dx, dg.to(g.dtype), db.to(g.dtype)
    xf, df = x.float(), dy.float()
    xh = (xf - mean[..., None]) * rstd[..., None]
    gd = df * g.float()
    m1 = gd.mean(-1, keepdim=True)
    m2 = (gd * xh).mean(-1, keepdim=True)
    dx = rstd[..., None] * (gd - m1 - xh * m2)
    if dres is not None:
        dx = dx + dres.float()
    dg = (df * xh).reshape(-1, H).sum(0)
    db = df.reshape(-1, H).sum(0)
    return dx.to(x.dtype), dg.to(g.dtype), db.to(g.dtype)


@layer_norm_bwd.register_fake
def _(dy, x, g, mean, rstd, dres):
    return torch.empty_like(x), torch.empty_like(g), torch.empty_like(g)


def _ln_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)  # unused outputs yield None, not a zero tensor + add
    x, g, b, eps = inputs
    _, mean, rstd = output
    ctx.save_for_backward(x, g, mean, rstd)


def _ln_bwd(ctx, dy, dmean, drstd):
    if dy is None:
        return None, None, None, None
    x, g, mean, rstd = ctx.saved_tensors
    dx, dg, db = layer_norm_bwd(dy, x, g, mean, rstd, None)
    return dx, dg, db, None


layer_norm.register_autograd(_ln_bwd, setup_context=_ln_setup)


def _aln_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)  # unused outputs yield None, not a zero tensor + add
    x, r, g, b, eps = inputs
    _, s, mean, rstd = output
    ctx.save_for_backward(s, g, mean, rstd)


def _aln_bwd(ctx, dy, ds, dmean, drstd):
    s, g, mean, rstd = ctx.saved_tensors
    if dy is None:
        return ds, ds, None, None, None
    dx, dg, db = layer_norm_bwd(dy, s, g, mean, rstd, ds)
    return dx, dx, dg, db, None


add_layer_norm.register_autograd(_aln_bwd, setup_context=_aln_setup)


# ---- RMSNorm: the LayerNorm kernels' `rms` variant (no mean, no beta): y = x * rstd * g, rstd = rsqrt(mean(x^2) + eps)
def _rms_ref(x: Tensor, g: Tensor, eps: float):
    xf = x.float()
    rstd = torch.rsqrt(xf.pow(2).mean(-1) + eps)
    return (xf * rstd[..., None] * g.float()).to(x.dtype), rstd


@torch.library.custom_op("alpa_b200::rms_norm", mutates_args=())
def rms_norm(x: Tensor, g: Tensor, eps: float) -> Tuple[Tensor, Tensor]:
    """(y, rstd); rstd is fp32 with shape x.shape[:-1]."""
    if C := _kernels("rms_norm", x, g, unsupported=_ln_unsupported(x.shape[-1])):
        y, _, rstd, _ = C.layernorm_fwd(x.contiguous(), None, g, None, eps, False, rms=True)
        return y, rstd.view(x.shape[:-1])
    return _rms_ref(x, g, eps)


@rms_norm.register_fake
def _(x, g, eps):
    return torch.empty_like(x), x.new_empty(x.shape[:-1], dtype=torch.float32)


@torch.library.custom_op("alpa_b200::add_rms_norm", mutates_args=())
def add_rms_norm(x: Tensor, r: Tensor, g: Tensor, eps: float) -> Tuple[Tensor, Tensor, Tensor]:
    """s = x + r (rounded to x's dtype); (rms_norm(s), s, rstd) in one pass."""
    if C := _kernels("add_rms_norm", x, r, g, unsupported=_ln_unsupported(x.shape[-1])):
        y, _, rstd, s = C.layernorm_fwd(x.contiguous(), r.contiguous(), g, None, eps, True, rms=True)
        return y, s, rstd.view(x.shape[:-1])
    s = x + r
    y, rstd = _rms_ref(s, g, eps)
    return y, s, rstd


@add_rms_norm.register_fake
def _(x, r, g, eps):
    return torch.empty_like(x), torch.empty_like(x), x.new_empty(x.shape[:-1], dtype=torch.float32)


@torch.library.custom_op("alpa_b200::rms_norm_bwd", mutates_args=())
def rms_norm_bwd(dy: Tensor, x: Tensor, g: Tensor, rstd: Tensor, dres: Optional[Tensor]) -> Tuple[Tensor, Tensor]:
    """(dx [+ dres], dgamma) of y = rms_norm(x): dx = rstd * (g*dy - xhat * mean(g*dy*xhat)), xhat = x * rstd."""
    H = x.shape[-1]
    if C := _kernels("rms_norm_bwd", dy, x, g, unsupported=_ln_unsupported(H)):
        dg = torch.zeros(H, device=x.device, dtype=torch.float32)
        dx = C.layernorm_bwd(dy.contiguous(), x.contiguous(), g, None, rstd.reshape(-1).contiguous(),
                             dres.contiguous() if dres is not None else None, dg, None, rms=True)
        return dx, dg.to(g.dtype)
    xf, df = x.float(), dy.float()
    xh = xf * rstd[..., None]
    gd = df * g.float()
    dx = rstd[..., None] * (gd - xh * (gd * xh).mean(-1, keepdim=True))
    if dres is not None:
        dx = dx + dres.float()
    dg = (df * xh).reshape(-1, H).sum(0)
    return dx.to(x.dtype), dg.to(g.dtype)


@rms_norm_bwd.register_fake
def _(dy, x, g, rstd, dres):
    return torch.empty_like(x), torch.empty_like(g)


def _rms_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)  # unused outputs yield None, not a zero tensor + add
    x, g, eps = inputs
    ctx.save_for_backward(x, g, output[1])


def _rms_bwd(ctx, dy, drstd):
    if dy is None:
        return None, None, None
    x, g, rstd = ctx.saved_tensors
    dx, dg = rms_norm_bwd(dy, x, g, rstd, None)
    return dx, dg, None


rms_norm.register_autograd(_rms_bwd, setup_context=_rms_setup)


def _arms_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)  # unused outputs yield None, not a zero tensor + add
    x, r, g, eps = inputs
    _, s, rstd = output
    ctx.save_for_backward(s, g, rstd)


def _arms_bwd(ctx, dy, ds, drstd):
    s, g, rstd = ctx.saved_tensors
    if dy is None:
        return ds, ds, None, None
    dx, dg = rms_norm_bwd(dy, s, g, rstd, ds)
    return dx, dx, dg, None


add_rms_norm.register_autograd(_arms_bwd, setup_context=_arms_setup)


# =================================================================================================
# attention: q, k, v are [B, S, heads, D]
# =================================================================================================
def _attn_ref(q, k, v, scale, causal):
    qf, kf, vf = (t.float().permute(0, 2, 1, 3) for t in (q, k, v))
    s = torch.matmul(qf, kf.transpose(-1, -2)) * scale
    if causal:
        Sq, Sk = s.shape[-2:]
        mask = torch.ones(Sq, Sk, device=s.device, dtype=torch.bool).tril(Sk - Sq)
        s = s.masked_fill(~mask, float("-inf"))
    lse = torch.logsumexp(s, dim=-1)
    p = torch.exp(s - _finite_lse(lse)[..., None])
    o = torch.matmul(p, vf).permute(0, 2, 1, 3)
    return o.to(q.dtype).contiguous(), lse


def _finite_lse(lse):
    """lse with the -inf of rows that see no key replaced by 0: exp(s - lse) is then exp(-inf) = 0 on those rows, so
    they get O = 0 and zero gradients (as the native kernels give) instead of exp(-inf + inf) = NaN."""
    return lse.masked_fill(lse == float("-inf"), 0.0)


def _attn_unsupported(D: int, stride: int = 1) -> Optional[str]:
    """Why the sm_90a attention kernels cannot take head dim D at element stride `stride` (they need a contiguous
    multiple of 8 up to 128), or None."""
    if D % 8 or D > 128:
        return "head dim not a multiple of 8 up to 128"
    return None if stride == 1 else "head dim not contiguous"


@torch.library.custom_op("alpa_b200::attention", mutates_args=())
def attention(q: Tensor, k: Tensor, v: Tensor, scale: float, causal: bool) -> Tuple[Tensor, Tensor]:
    """(o [B,S,h,D], lse [B,h,S]) = softmax(q k^T * scale [+ causal mask]) v.  A grouped q [B,S,Hkv,G,D] against k / v
    [B,S,Hkv,D] (query head kv * G + g uses K/V head kv) gives o [B,S,Hkv,G,D] and lse [B,Hkv,G,S]."""
    if C := _kernels("attention", q, k, v, unsupported=_attn_unsupported(q.shape[-1], q.stride(-1))):
        o, lse = C.attention_fwd(q, k, v, scale, causal)
        return o, lse
    if q.dim() == 5:
        return _gqa_attn_ref(q, k, v, scale, causal)
    return _attn_ref(q, k, v, scale, causal)


@attention.register_fake
def _(q, k, v, scale, causal):
    if q.dim() == 5:
        B, S, Hkv, G, D = q.shape
        return q.new_empty(B, S, Hkv, G, D), q.new_empty(B, Hkv, G, S, dtype=torch.float32)
    B, S, H, D = q.shape
    return q.new_empty(B, S, H, D), q.new_empty(B, H, S, dtype=torch.float32)


@torch.library.custom_op("alpa_b200::attention_bwd", mutates_args=())
def attention_bwd(do: Tensor, q: Tensor, k: Tensor, v: Tensor, o: Tensor, lse: Tensor, scale: float,
                  causal: bool) -> Tuple[Tensor, Tensor, Tensor]:
    if C := _kernels("attention_bwd", do, q, k, v, o, unsupported=_attn_unsupported(q.shape[-1], q.stride(-1))):
        dq, dk, dv = C.attention_bwd(do, q, k, v, o, lse, scale, causal)
        return dq, dk, dv
    if q.dim() == 5:
        return _gqa_attn_ref_bwd(do, q, k, v, o, lse, scale, causal)
    return _attn_ref_bwd(do, q, k, v, o, lse, scale, causal)


@attention_bwd.register_fake
def _(do, q, k, v, o, lse, scale, causal):
    return (q.new_empty(q.shape), k.new_empty(k.shape), v.new_empty(v.shape))


def _attn_ref_bwd(do, q, k, v, o, lse, scale, causal):
    """Gradients of `_attn_ref`."""
    qf, kf, vf = (t.float().permute(0, 2, 1, 3) for t in (q, k, v))
    dof = do.float().permute(0, 2, 1, 3)
    of = o.float().permute(0, 2, 1, 3)
    s = torch.matmul(qf, kf.transpose(-1, -2)) * scale
    if causal:
        Sq, Sk = s.shape[-2:]
        mask = torch.ones(Sq, Sk, device=s.device, dtype=torch.bool).tril(Sk - Sq)
        s = s.masked_fill(~mask, float("-inf"))
    p = torch.exp(s - _finite_lse(lse)[..., None])
    dv = torch.matmul(p.transpose(-1, -2), dof)
    dp = torch.matmul(dof, vf.transpose(-1, -2))
    delta = (dof * of).sum(-1, keepdim=True)
    ds = p * (dp - delta) * scale
    dq = torch.matmul(ds, kf)
    dk = torch.matmul(ds.transpose(-1, -2), qf)
    return tuple(t.permute(0, 2, 1, 3).contiguous().to(q.dtype) for t in (dq, dk, dv))


def _attn_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)  # unused outputs yield None, not a zero tensor + add
    q, k, v, scale, causal = inputs
    o, lse = output
    ctx.save_for_backward(q, k, v, o, lse)
    ctx.scale, ctx.causal = scale, causal


def _attn_bwd(ctx, do, dlse):
    if do is None:
        return None, None, None, None, None
    q, k, v, o, lse = ctx.saved_tensors
    dq, dk, dv = attention_bwd(do, q, k, v, o, lse, ctx.scale, ctx.causal)
    return dq, dk, dv, None, None


attention.register_autograd(_attn_bwd, setup_context=_attn_setup)


# ---- packed variant: qkv is one [B, S, kv_heads, G + 2, D] tensor, a view of the fused QKV projection whose output
# features are ordered (K/V head, {its G query heads, k, v}, D): slots 0..G-1 are the query heads kv * G + g of K/V head
# kv, slot G its K and slot G + 1 its V (HF's repeat_kv order).  A contiguous split of the feature dim is then a split
# over K/V heads that never splits a group (the Megatron layout); G = 1 is multi-head attention, features ordered
# (head, {q, k, v}, D).  Forward and backward touch the projection output / gradient in place: no split/concat copies.
def _gqa_split(qkv):
    G = qkv.shape[3] - 2
    return qkv[:, :, :, :G], qkv[:, :, :, G], qkv[:, :, :, G + 1]


def _gqa_expand(q, k, v):
    """q [B,Sq,Hkv,G,D], k / v [B,Skv,Hkv,D] -> [B,S,Hkv*G,D] each, K/V repeated per query head."""
    B, Sq, Hkv, G, D = q.shape
    rep = lambda t: t[:, :, :, None].expand(-1, -1, -1, G, -1).reshape(B, t.shape[1], Hkv * G, D)  # noqa: E731
    return q.reshape(B, Sq, Hkv * G, D), rep(k), rep(v)


def _gqa_attn_ref(q, k, v, scale, causal):
    """PyTorch grouped-query attention: q [B,Sq,Hkv,G,D], k / v [B,Skv,Hkv,D] -> (o [B,Sq,Hkv,G,D], lse [B,Hkv,G,Sq]).
    Rows that see no key give O = 0, as in `_attn_ref`."""
    B, Sq, Hkv, G, D = q.shape
    o, lse = _attn_ref(*_gqa_expand(q, k, v), scale, causal)
    return o.view(B, Sq, Hkv, G, D), lse.view(B, Hkv, G, Sq)


def _gqa_attn_ref_bwd(do, q, k, v, o, lse, scale, causal):
    """Gradients of `_gqa_attn_ref`: dq like q, dk / dv like k / v (summed over each group in fp32)."""
    B, Sq, Hkv, G, D = q.shape
    Hq = Hkv * G
    dq, dk, dv = _attn_ref_bwd(do.reshape(B, Sq, Hq, D), *_gqa_expand(q, k, v), o.reshape(B, Sq, Hq, D),
                               lse.reshape(B, Hq, Sq), scale, causal)
    group_sum = lambda t: t.view(B, -1, Hkv, G, D).float().sum(3).to(q.dtype)  # noqa: E731
    return dq.view(B, Sq, Hkv, G, D), group_sum(dk), group_sum(dv)


@torch.library.custom_op("alpa_b200::attention_gqa_packed", mutates_args=())
def attention_gqa_packed(qkv: Tensor, scale: float, causal: bool) -> Tuple[Tensor, Tensor]:
    """(o [B,S,Hkv,G,D], lse [B,Hkv,G,S]) = grouped-query softmax attention of qkv [B,S,Hkv,G+2,D].  G = 1 is
    multi-head attention."""
    q, k, v = _gqa_split(qkv)
    D = qkv.shape[-1]
    if C := _kernels("attention_gqa_packed", qkv,
                     unsupported=_attn_unsupported(D, qkv.stride(-1)) or (None if q.shape[3] else "empty query group")):
        o, lse = C.attention_fwd(q, k, v, scale, causal)
        return o, lse
    return _gqa_attn_ref(q, k, v, scale, causal)


@attention_gqa_packed.register_fake
def _(qkv, scale, causal):
    B, S, Hkv, P, D = qkv.shape
    return qkv.new_empty(B, S, Hkv, P - 2, D), qkv.new_empty(B, Hkv, P - 2, S, dtype=torch.float32)


@torch.library.custom_op("alpa_b200::attention_gqa_packed_bwd", mutates_args=())
def attention_gqa_packed_bwd(do: Tensor, qkv: Tensor, o: Tensor, lse: Tensor, scale: float, causal: bool) -> Tensor:
    """dqkv [B,S,Hkv,G+2,D]: dQ in slots 0..G-1, dK (summed over the group) in slot G, dV in slot G + 1"""
    q, k, v = _gqa_split(qkv)
    G, D = q.shape[3], qkv.shape[-1]
    dqkv = torch.empty(qkv.shape, device=qkv.device, dtype=qkv.dtype)
    if C := _kernels("attention_gqa_packed_bwd", qkv, do, o,
                     unsupported=_attn_unsupported(D, qkv.stride(-1)) or (None if G else "empty query group")):
        C.attention_bwd(do, q, k, v, o, lse, scale, causal, dqkv[:, :, :, :G], dqkv[:, :, :, G], dqkv[:, :, :, G + 1])
        return dqkv
    dqkv[:, :, :, :G], dqkv[:, :, :, G], dqkv[:, :, :, G + 1] = _gqa_attn_ref_bwd(do, q, k, v, o, lse, scale, causal)
    return dqkv


@attention_gqa_packed_bwd.register_fake
def _(do, qkv, o, lse, scale, causal):
    return torch.empty_like(qkv)


def _attn_packed_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)  # unused outputs yield None, not a zero tensor + add
    qkv, scale, causal = inputs
    o, lse = output
    ctx.save_for_backward(qkv, o, lse)
    ctx.scale, ctx.causal = scale, causal


def _attn_gqa_bwd(ctx, do, dlse):
    if do is None:
        return None, None, None
    qkv, o, lse = ctx.saved_tensors
    return attention_gqa_packed_bwd(do, qkv, o, lse, ctx.scale, ctx.causal), None, None


attention_gqa_packed.register_autograd(_attn_gqa_bwd, setup_context=_attn_packed_setup)


# ---- rotary position embedding on the packed [B, S, Hkv, G + 2, D] tensor (HF's rotate_half convention): slots 0..G
# (the query heads and K) rotate, slot G + 1 (V) passes through.  Element i pairs with i + D/2 at angle
# float(position) * inv_freq[i], inv_freq = 1 / theta ** (arange(0, D, 2) / D) as HF builds it.
@cache
def _inv_freq(D: int, theta: float, device: str) -> Tensor:
    """HF's default rope frequencies, computed on the CPU as HF does and cached per (D, theta, device)."""
    return (1.0 / (theta ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))).to(device)


def _rotary_ref(qkv: Tensor, position_ids: Tensor, inv_freq: Tensor, inverse: bool) -> Tensor:
    D, R = qkv.shape[-1], qkv.shape[3] - 1
    ang = position_ids.float()[..., None] * inv_freq                  # [B, S, D/2], the fp32 product HF forms
    c, s = ang.cos()[:, :, None, None], ang.sin()[:, :, None, None]
    if inverse:
        s = -s
    x = qkv[:, :, :, :R].float()
    x1, x2 = x[..., :D // 2], x[..., D // 2:]
    rot = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1).to(qkv.dtype)
    return torch.cat([rot, qkv[:, :, :, R:]], 3)


def _rotary_unsupported(qkv: Tensor) -> Optional[str]:
    """Why the rotary kernel (8 elements of each half per vector) cannot take qkv, or None."""
    if qkv.shape[-1] % 16:
        return "head dim not a multiple of 16"
    return None if qkv.is_contiguous() and qkv.data_ptr() % 16 == 0 else "packed qkv not contiguous"


@torch.library.custom_op("alpa_b200::rotary_packed", mutates_args=())
def rotary_packed(qkv: Tensor, position_ids: Tensor, theta: float, inverse: bool) -> Tensor:
    """qkv [B,S,Hkv,G+2,D] with the G query heads and K of every K/V head rotated by position_ids (by minus the angle
    when `inverse`, which is the backward); V copied.  position_ids: integer, [B, S] or broadcastable to it (HF's
    [1, S]), on qkv's device."""
    inv_freq = _inv_freq(qkv.shape[-1], float(theta), str(qkv.device))
    if C := _kernels("rotary_packed", qkv, position_ids, unsupported=lambda: _rotary_unsupported(qkv)):
        pos = position_ids.to(torch.int64).expand(qkv.shape[0], qkv.shape[1]).contiguous()
        return C.rotary_packed(qkv, pos, inv_freq, inverse)
    return _rotary_ref(qkv, position_ids, inv_freq, inverse)


@rotary_packed.register_fake
def _(qkv, position_ids, theta, inverse):
    return torch.empty_like(qkv)


def _rotary_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)  # unused outputs yield None, not a zero tensor + add
    _, position_ids, theta, inverse = inputs
    ctx.save_for_backward(position_ids)
    ctx.theta, ctx.inverse = theta, inverse


def _rotary_bwd(ctx, dy):
    if dy is None:
        return None, None, None, None
    (position_ids,) = ctx.saved_tensors
    return rotary_packed(dy, position_ids, ctx.theta, not ctx.inverse), None, None, None


rotary_packed.register_autograd(_rotary_bwd, setup_context=_rotary_setup)


# ---- SwiGLU on interleaved pairs: gu [..., I, 2] holds (gate j, up j) at fc1 output features (2j, 2j + 1), so a
# contiguous column split of fc1 keeps every pair on one device.
def _swiglu_unsupported(*ts: Tensor) -> Optional[str]:
    """Why the SwiGLU kernels (4 pairs per 16-byte vector) cannot take these operands, or None."""
    if ts[-1].shape[-2] % 4:
        return "I not a multiple of 4"
    return None if all(t.is_contiguous() and t.data_ptr() % 16 == 0 for t in ts) else "operands not contiguous"


@torch.library.custom_op("alpa_b200::swiglu", mutates_args=())
def swiglu(gu: Tensor) -> Tensor:
    """h [..., I] = silu(gu[..., 0]) * gu[..., 1]"""
    if C := _kernels("swiglu", gu, unsupported=lambda: _swiglu_unsupported(gu)):
        return C.swiglu_fwd(gu)
    g, u = gu.float().unbind(-1)
    return (F.silu(g) * u).to(gu.dtype)


@swiglu.register_fake
def _(gu):
    return gu.new_empty(gu.shape[:-1])


@torch.library.custom_op("alpa_b200::swiglu_bwd", mutates_args=())
def swiglu_bwd(dh: Tensor, gu: Tensor) -> Tensor:
    """dgu [..., I, 2] = (dh * u * s (1 + g (1 - s)), dh * silu(g)), s = sigmoid(g): recomputed from gu."""
    if C := _kernels("swiglu_bwd", dh, gu, unsupported=lambda: _swiglu_unsupported(dh[..., None], gu)):
        return C.swiglu_bwd(dh, gu)
    g, u = gu.float().unbind(-1)
    d = dh.float()
    s = torch.sigmoid(g)
    return torch.stack([d * u * s * (1 + g * (1 - s)), d * g * s], -1).to(gu.dtype)


@swiglu_bwd.register_fake
def _(dh, gu):
    return torch.empty_like(gu)


def _swiglu_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)  # unused outputs yield None, not a zero tensor + add
    ctx.save_for_backward(inputs[0])


def _swiglu_grad(ctx, dh):
    if dh is None:
        return None
    (gu,) = ctx.saved_tensors
    return swiglu_bwd(dh, gu)


swiglu.register_autograd(_swiglu_grad, setup_context=_swiglu_setup)

# =================================================================================================
# embedding (token gather [+ position]) -- the reference lowers this to a one-hot matmul
# (alpa/monkey_patch.py:241-261) to make the vocab dim shardable; we keep a real gather and give the
# planner a vocab-parallel (masked gather + all-reduce) strategy instead.
# =================================================================================================
@torch.library.custom_op("alpa_b200::embedding", mutates_args=())
def embedding(ids: Tensor, wte: Tensor, vocab_start: int = 0) -> Tensor:
    """x[..., H] = wte[ids - vocab_start] (zeros for ids outside this vocab shard)"""
    V = wte.shape[0]
    if C := _kernels("embedding", wte, unsupported=None if wte.shape[1] % 8 == 0 else "H not a multiple of 8"):
        return C.embedding_fwd(ids.contiguous(), None, wte.contiguous(), None, vocab_start)
    local = ids - vocab_start
    ok = (local >= 0) & (local < V)
    out = F.embedding(local.clamp(0, V - 1), wte)
    return out * ok[..., None].to(out.dtype)      # rows outside this vocabulary shard contribute zeros


@embedding.register_fake
def _(ids, wte, vocab_start=0):
    return wte.new_empty(*ids.shape, wte.shape[1])


@torch.library.custom_op("alpa_b200::embedding_bwd", mutates_args=())
def embedding_bwd(ids: Tensor, dy: Tensor, num_rows: int, vocab_start: int = 0) -> Tensor:
    """dwte[num_rows, H] = scatter-add of dy rows at (ids - vocab_start)"""
    H = dy.shape[-1]
    if C := _kernels("embedding_bwd", dy, unsupported=None if H % 2 == 0 else "odd H"):
        dt = torch.zeros(num_rows, H, device=dy.device, dtype=torch.float32)
        C.embedding_bwd_(ids.contiguous(), dy.contiguous(), dt, vocab_start)
        return dt.to(dy.dtype)
    local = (ids - vocab_start).reshape(-1)
    ok = (local >= 0) & (local < num_rows)
    d2 = dy.reshape(-1, H).float() * ok[:, None].float()
    out = torch.zeros(num_rows, H, device=dy.device, dtype=torch.float32)
    out.index_add_(0, local.clamp(0, num_rows - 1), d2)
    return out.to(dy.dtype)


@embedding_bwd.register_fake
def _(ids, dy, num_rows, vocab_start=0):
    return dy.new_empty(num_rows, dy.shape[-1])


def _emb_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)  # unused outputs yield None, not a zero tensor + add
    ids, wte, vocab_start = inputs
    ctx.save_for_backward(ids)
    ctx.num_rows = wte.shape[0]
    ctx.vocab_start = vocab_start


def _emb_bwd(ctx, dy):
    if dy is None:
        return None, None, None
    (ids,) = ctx.saved_tensors
    return None, embedding_bwd(ids, dy, ctx.num_rows, ctx.vocab_start), None


embedding.register_autograd(_emb_bwd, setup_context=_emb_setup)


# =================================================================================================
# fp8 KV cache (serving): e4m3 rows with one fp32 scale per (token, K/V head)
# =================================================================================================
class Fp8KV:
    """One K or V cache in fp8: `data` e4m3 [B, S, Hkv, D] with `scale` fp32 [B, Hkv, S], or the slot-addressed
    `data` [slots, Hkv, D] with `scale` [Hkv, slots].  A row x of D bf16 values is stored as
        s = max(amax(|x|), 1e-8) / 448,   q = e4m3_rne(x / s)    (both divisions correctly rounded)
    and reads back as float(q) * s.  The scales are head-major so that the consecutive keys a decode CTA reads share
    their sectors.  The serving ops (decode / ragged attention, `kv_cache_store`, `kv_cache_load`) take an Fp8KV where
    they take a bf16 cache tensor; the batch slicing and the `index_select` / `copy_` reordering that generation
    applies to cache tensors work on it too (4-D caches), moving data and scales together."""
    __slots__ = ("data", "scale")

    def __init__(self, data: Tensor, scale: Tensor):
        self.data, self.scale = data, scale

    @classmethod
    def zeros(cls, shape, device) -> "Fp8KV":
        """An all-zero cache of data shape [B, S, Hkv, D] or [slots, Hkv, D]."""
        *lead, S, H, _ = shape
        return cls(torch.zeros(shape, dtype=torch.float8_e4m3fn, device=device),
                   torch.zeros(*lead, H, S, dtype=torch.float32, device=device))

    def _batched(self):
        if self.data.dim() != 4:
            raise TypeError("batch indexing needs a [B, S, Hkv, D] cache")

    def __getitem__(self, idx) -> "Fp8KV":
        self._batched()
        if not isinstance(idx, slice):
            raise TypeError("Fp8KV supports slicing along the batch only")
        return Fp8KV(self.data[idx], self.scale[idx])

    def index_select(self, dim: int, index: Tensor) -> "Fp8KV":
        self._batched()
        if dim != 0:
            raise ValueError("Fp8KV reorders along the batch (dim 0) only")
        return Fp8KV(self.data.view(torch.uint8).index_select(0, index).view(torch.float8_e4m3fn),
                     self.scale.index_select(0, index))

    def copy_(self, other: "Fp8KV") -> "Fp8KV":
        self.data.view(torch.uint8).copy_(other.data.view(torch.uint8))
        self.scale.copy_(other.scale)
        return self

    def nbytes(self) -> int:
        return self.data.numel() + self.scale.numel() * 4

    def values(self, end: Optional[int] = None) -> Tensor:
        """The fp32 values float(q) * s ([B, end, Hkv, D] of rows [0, end), or [slots, Hkv, D])."""
        if self.data.dim() == 3:
            return self.data.float() * self.scale.t()[..., None]
        return self.data[:, :end].float() * self.scale[:, :, :end].transpose(1, 2)[..., None]


_KV_DTYPES = (torch.bfloat16, torch.float8_e4m3fn)


def kv_cache_nbytes(cache) -> int:
    """Bytes held by a model's KV cache: a list of (k, v) bf16 tensors or Fp8KV pairs."""
    return sum(t.nbytes() if isinstance(t, Fp8KV) else t.numel() * t.element_size() for kv in cache for t in kv)


def _kv_quant_ref(x: Tensor) -> Tuple[Tensor, Tensor]:
    """(q e4m3 [..., D], s fp32 [...]) of rows x [..., D] in the Fp8KV format.  Both divisions are tensor by tensor:
    PyTorch divides by a Python scalar as a multiply by its reciprocal on CUDA, which is not correctly rounded."""
    xf = x.float()
    amax = xf.abs().amax(-1).clamp(min=1e-8)
    s = amax / torch.full_like(amax, 448.0)
    return (xf / s[..., None]).to(torch.float8_e4m3fn), s


def _kv_store_ref(k: Tensor, v: Tensor, k_cache: Fp8KV, v_cache: Fp8KV, start: int, rows: Optional[Tensor]):
    B, T, H, D = k.shape
    for x, c in ((k, k_cache), (v, v_cache)):
        q, sc = _kv_quant_ref(x)
        q8 = q.view(torch.uint8)
        if rows is None:
            c.data.view(torch.uint8)[:B, start:start + T] = q8
            c.scale[:B, :, start:start + T] = sc.transpose(1, 2)
        else:
            c.data.view(torch.uint8)[rows] = q8.reshape(B * T, H, D)
            c.scale[:, rows] = sc.reshape(B * T, H).t()


def _kv_store_unsupported(k: Tensor, v: Tensor) -> Optional[str]:
    """Why the store kernel (one warp per row, 16-byte loads of 8 channels) cannot take k / v, or None."""
    D = k.shape[-1]
    if D % 8 or D > 256:
        return "head dim not a multiple of 8 up to 256"
    for x in (k, v):
        if x.stride(-1) != 1 or any(st % 8 for st in x.stride()[:-1]) or x.data_ptr() % 16:
            return "K / V rows not 16-byte aligned"
    return None


def kv_cache_store(k: Tensor, v: Tensor, k_cache: Fp8KV, v_cache: Fp8KV, start: int = 0,
                   rows: Optional[Tensor] = None) -> None:
    """Quantise bf16 K / V rows into fp8 caches.  k / v: [B, T, Hkv, D] views, each with its own strides (the packed
    QKV projection's K and V slots, or a rotated K next to the V slot, are fine).  For [B, S, Hkv, D] caches token
    (b, t) goes to row start + t of sequence b; for slot-addressed [slots, Hkv, D] caches `rows` (int64 [B * T]) gives
    each token's slot.  The slots must lie inside the cache: the kernel reads them on the device only and writes
    nothing for a slot outside it."""
    if (rows is None) != (k_cache.data.dim() == 4):
        raise ValueError("kv_cache_store: [B, S, Hkv, D] caches take `start`, slot-addressed caches take `rows`")
    if C := _kernels("kv_cache_store", k, v, k_cache.data, v_cache.data, dtypes=_KV_DTYPES,
                     unsupported=lambda: _kv_store_unsupported(k, v)):
        C.kv_cache_store(k, v, k_cache.data, v_cache.data, k_cache.scale, v_cache.scale, start, rows)
        return
    _kv_store_ref(k, v, k_cache, v_cache, start, rows)


def kv_cache_load(cache: Fp8KV, end: int) -> Tensor:
    """Rows [0, end) of an fp8 [B, S, Hkv, D] cache dequantised to bf16 [B, end, Hkv, D]: bf16(float(q) * s).  The
    scratch the prefill's attention reads."""
    D = cache.data.shape[-1]
    if C := _kernels("kv_cache_load", cache.data, dtypes=_KV_DTYPES,
                     unsupported=None if D % 8 == 0 else "head dim not a multiple of 8"):
        return C.kv_cache_load(cache.data, cache.scale, end)
    return cache.values(end).to(torch.bfloat16)


def _kv_pair(k_cache, v_cache):
    """(k data, v data, dtypes the kernels admit, scale kwargs) of a bf16 or Fp8KV cache pair."""
    if isinstance(k_cache, Fp8KV):
        return k_cache.data, v_cache.data, _KV_DTYPES, {"k_scale": k_cache.scale, "v_scale": v_cache.scale}
    return k_cache, v_cache, (torch.bfloat16,), {}


def _decode_fp8_unsupported(D: int, k_cache) -> Optional[str]:
    """Why the fp8 decode kernel cannot take head dim D (8-byte row pieces of 8 channels, up to 128), or None."""
    if not isinstance(k_cache, Fp8KV) or (D % 8 == 0 and D <= 128):
        return None
    return "head dim not a multiple of 8 up to 128"


# =================================================================================================
# decode attention over a KV cache whose valid length lives on the device (serving; not differentiable)
# =================================================================================================
def decode_attention(q: Tensor, k_new: Tensor, v_new: Tensor, k_cache: Tensor, v_cache: Tensor, kv_len: Tensor,
                     scale: float) -> Tensor:
    """One new token per sequence with the cache append fused in.  q / k_new / v_new: [B, 1, h, D] (views of the fused
    QKV projection are fine); k/v_cache: [B, S_max, h, D], updated in place at row kv_len-1; kv_len: int32 scalar tensor
    = valid rows including the new one; because it is read on the device, one captured CUDA graph serves every decode
    position.  Returns o [B, 1, h, D].  One cache-streaming kernel: no separate cache copies, no padded tensor-core
    attention.  With Fp8KV caches the new rows are quantised as they are appended and every query attends to the
    cache's values float(q) * s, its own token's included."""
    kd, vd, dtypes, scales = _kv_pair(k_cache, v_cache)
    if C := _kernels("decode_attention", q, kd, vd, dtypes=dtypes,
                     unsupported=lambda: _decode_fp8_unsupported(q.shape[-1], k_cache)):
        if k_new.stride() != v_new.stride() or k_new.stride(-1) != 1:      # e.g. k went through rotary, v did not
            k_new, v_new = k_new.contiguous(), v_new.contiguous()
        return C.decode_attention(q if q.stride(-1) == 1 else q.contiguous(), k_new, v_new, kd, vd, kv_len,
                                  scale, **scales)
    n = int(kv_len)
    if scales:
        _kv_store_ref(k_new, v_new, k_cache, v_cache, n - 1, None)
        return _attn_ref(q, k_cache.values(n), v_cache.values(n), scale, True)[0]
    k_cache[:, n - 1:n] = k_new
    v_cache[:, n - 1:n] = v_new
    return _attn_ref(q, k_cache[:, :n], v_cache[:, :n], scale, True)[0]


def _decode_gqa_unsupported(qkv_new: Tensor) -> Optional[str]:
    """Why the decode kernel's packed form cannot take qkv_new [B, 1, Hkv, G + 2, D], or None: it reads each head's D
    channels and their rotary partners 16 bytes at a time from one contiguous row."""
    D = qkv_new.shape[-1]
    if D % 16 or D > 128:
        return "head dim not a multiple of 16 up to 128"
    return None if qkv_new.is_contiguous() and qkv_new.data_ptr() % 16 == 0 else "packed row not contiguous"


def decode_attention_gqa(qkv_new: Tensor, k_cache: Tensor, v_cache: Tensor, kv_len: Tensor,
                         position_ids: Optional[Tensor], scale: float, theta: float = 10000.0) -> Tensor:
    """Grouped-query decode step over the packed QKV row of the new token, qkv_new [B, 1, Hkv, G + 2, D] (the QKV
    projection's output: per K/V head its G query heads, k, v).  With `position_ids` (int64 [B, 1] on the device) the
    query heads and k are first rotated as `rotary_packed(qkv_new, position_ids, theta, False)` rotates them, bit for
    bit; None = no rotary.  The (rotated) k and v are appended to k/v_cache [B, S_max, Hkv, D] at row kv_len - 1
    (kv_len: int32 device scalar, valid rows including the new one), then query head kv * G + g attends to rows
    [0, kv_len) of K/V head kv.  One kernel launch that reads every cache row once for its whole group; one captured
    CUDA graph serves every position.  Returns o [B, 1, Hkv * G, D].  Fp8KV caches: see `decode_attention`."""
    B, _, Hkv, P, D = qkv_new.shape
    rope = position_ids is not None
    inv_freq = _inv_freq(D, float(theta), str(qkv_new.device)) if rope else None
    kd, vd, dtypes, scales = _kv_pair(k_cache, v_cache)
    if C := _kernels("decode_attention_gqa", qkv_new, kd, vd, dtypes=dtypes,
                     unsupported=lambda: _decode_gqa_unsupported(qkv_new)):
        pos = position_ids.to(torch.int64).reshape(B, 1).contiguous() if rope else None
        return C.decode_attention_packed(qkv_new, kd, vd, kv_len, scale, pos, inv_freq, **scales)
    if rope:
        qkv_new = _rotary_ref(qkv_new, position_ids, inv_freq, False)
    q, k, v = _gqa_split(qkv_new)
    n = int(kv_len)
    if scales:
        _kv_store_ref(k, v, k_cache, v_cache, n - 1, None)
        o, _ = _gqa_attn_ref(q, k_cache.values(n), v_cache.values(n), scale, True)
        return o.reshape(B, 1, Hkv * (P - 2), D)
    k_cache[:, n - 1:n] = k
    v_cache[:, n - 1:n] = v
    o, _ = _gqa_attn_ref(q, k_cache[:, :n], v_cache[:, :n], scale, True)
    return o.reshape(B, 1, Hkv * (P - 2), D)


# =================================================================================================
# traceable attention over a KV cache (functional: returns the appended caches) -- the op `@parallelize` sees when a
# decoder with a cache goes through the ILP / the inference pipeline (reference: examples/llm_serving/model/
# opt_model.py:283-330, the `cache_vector` update + attention of `OPTSelfAttention.__call__`)
# =================================================================================================
@torch.library.custom_op("alpa_b200::attention_cached", mutates_args=())
def attention_cached(q: Tensor, k_new: Tensor, v_new: Tensor, k_cache: Tensor, v_cache: Tensor, cache_len: Tensor,
                     scale: float) -> Tuple[Tensor, Tensor, Tensor]:
    """(o [B,T,h,D], k_cache' , v_cache') : append the T new key / value rows at cache rows cache_len .. cache_len+T-1
    and attend causally (query i sees rows 0 .. cache_len+i).  q / k_new / v_new: [B, T, h, D]; k/v_cache:
    [B, S_max, h, D]; cache_len: int32 scalar tensor read ON THE DEVICE, so one compiled executable (and one captured
    graph) serves every decode position.  Functional: the caches come back as new values; `attention_cached_`
    (used when the executable owns the cache buffers) appends in place."""
    k_out, v_out = k_cache.clone(), v_cache.clone()
    o = attention_cached_(q, k_new, v_new, k_out, v_out, cache_len, scale)
    return o, k_out, v_out


@attention_cached.register_fake
def _(q, k_new, v_new, k_cache, v_cache, cache_len, scale):
    return torch.empty_like(q, memory_format=torch.contiguous_format), torch.empty_like(k_cache), \
        torch.empty_like(v_cache)


def attention_cached_(q: Tensor, k_new: Tensor, v_new: Tensor, k_cache: Tensor, v_cache: Tensor, cache_len: Tensor,
                      scale: float) -> Tensor:
    """In-place form of `attention_cached`: k/v_cache are updated, o is returned."""
    T = q.shape[1]
    C = _kernels("attention_cached", q, k_cache, v_cache, unsupported=_attn_unsupported(q.shape[-1]))
    if C is not None and T == 1:
        return decode_attention(q, k_new, v_new, k_cache, v_cache, (cache_len.to(torch.int32) + 1).reshape(()), scale)
    # prompt chunk: same kernel path as the serving decoder's prefill (flash attention over the valid cache rows,
    # causal with Sq != Sk); the length is read on the host here -- only the T = 1 step has to be sync-free
    n0 = int(cache_len)
    k_cache[:, n0:n0 + T] = k_new
    v_cache[:, n0:n0 + T] = v_new
    k, v = k_cache[:, :n0 + T], v_cache[:, :n0 + T]
    if C is None:
        return _attn_ref(q, k, v, scale, True)[0]
    return attention(q if q.stride(-1) == 1 else q.contiguous(), k, v, scale, True)[0]       # the kernel reads D rows


# =================================================================================================
# attention of a ragged 1-D token batch over a slot-addressed KV cache (iteration-level batching; not differentiable)
# =================================================================================================
def ragged_attention(q: Tensor, k_cache: Tensor, v_cache: Tensor, seq_start: Tensor, ctx_len: Tensor, scale: float,
                     max_ctx: int, alibi: Optional[Tensor] = None, block_table: Optional[Tensor] = None,
                     block_size: Optional[int] = None) -> Tensor:
    """q: [T, h, D]; k/v_cache: [slots, h_kv, D] with h_kv dividing h (grouped-query attention: query head i reads
    cache head i // (h / h_kv)); token t attends to keys j < ctx_len[t] of its sequence (ctx_len 0 = padding token ->
    zeros).  Key j is cache row seq_start[t] + j, or with a paged cache (`block_table` int32 [N, max_blocks],
    `block_size` a power of two up to 1024) row block_table[seq_start[t], j // block_size] * block_size +
    j % block_size: seq_start then names the token's row of the table.  Table entries are not checked by the kernel
    (the block allocator builds them); the reference raises ValueError for an entry a token reads that lies outside
    the cache's blocks [0, (slots - 1) // block_size) (the last row is the scratch row).  Paged and contiguous calls on
    the same keys give the same bits.  `max_ctx` bounds ctx_len (sizes the score buffer).  `alibi`: optional fp32 [h]
    slopes, bias = slope * key position j.  Fp8KV caches ([slots, h_kv, D] data): tokens attend to the values
    float(q) * s.  (reference: the external fused_mmha of opt_model_1d.py:151-178)"""
    if (block_table is None) != (block_size is None):
        raise ValueError("ragged_attention: a paged cache needs both block_table and block_size")
    kd, vd, dtypes, scales = _kv_pair(k_cache, v_cache)
    if C := _kernels("ragged_attention", q, kd, vd, dtypes=dtypes,
                     unsupported=lambda: None if not scales or q.shape[-1] % 8 == 0 else "head dim not a multiple of 8"):
        paged = {} if block_table is None else {"block_table": block_table, "block_size": int(block_size)}
        return C.ragged_attention(q if q.stride(-1) == 1 else q.contiguous(), kd, vd, seq_start, ctx_len,
                                  scale, max_ctx, alibi, **scales, **paged)
    if scales:
        k_cache, v_cache = k_cache.values(), v_cache.values()
    T, h, D = q.shape
    longest = int(ctx_len.max()) if T else 0
    if longest > max_ctx:
        # the kernel's score buffer holds max_ctx keys; clamping would silently drop the newest keys
        raise ValueError(f"ragged_attention: ctx_len {longest} exceeds max_ctx {max_ctx}")
    n = longest
    if n == 0:
        return torch.zeros_like(q)
    j = torch.arange(n, device=q.device)
    valid = j[None, :] < ctx_len.long()[:, None]                                                 # [T, n]
    if block_table is None:
        idx = (seq_start.long()[:, None] + j[None, :]).clamp_(max=k_cache.shape[0] - 1)          # [T, n]
    else:
        bs = int(block_size)
        if bs < 1 or bs > 1024 or bs & (bs - 1) or block_table.shape[1] * bs < max_ctx:
            raise ValueError(f"ragged_attention: block size {bs} is not a power of two up to 1024, or "
                             f"{block_table.shape[1]} blocks per table row do not cover max_ctx {max_ctx}")
        rows = block_table.long()[seq_start.long()]                                              # [T, max_blocks]
        blk = rows.gather(1, (j // bs).clamp(max=rows.shape[1] - 1).expand(T, n))                # [T, n]
        nblk = (k_cache.shape[0] - 1) // bs
        bad = valid & ((blk < 0) | (blk >= nblk))
        if bool(bad.any()):
            raise ValueError(f"ragged_attention: block table entry {int(blk[bad][0])} lies outside the cache's "
                             f"{nblk} blocks")
        idx = torch.where(valid, blk * bs + j % bs, 0)
    G = h // k_cache.shape[1]
    k = k_cache[idx].float().repeat_interleave(G, dim=2)                                         # [T, n, h, D]
    v = v_cache[idx].float().repeat_interleave(G, dim=2)
    s = torch.einsum("thd,tnhd->thn", q.float() * scale, k)
    if alibi is not None:
        s = s + alibi.view(1, h, 1) * j.view(1, 1, n)
    s = s.masked_fill(~valid[:, None, :], float("-inf"))
    p = torch.softmax(s, dim=-1)
    p = torch.nan_to_num(p, nan=0.0)                                                             # padding rows
    return torch.einsum("thn,tnhd->thd", p, v).to(q.dtype)


def _paged_prefill_unsupported(q: Tensor, block_size: int) -> Optional[str]:
    """Why the paged prefill kernel cannot take these operands, or None."""
    if q.shape[-1] not in (64, 128):
        return "head dim not 64 or 128"
    if block_size < 16:
        return "block size under 16"
    if q.stride(-1) != 1 or any(s % 8 for s in q.stride()[:-1]) or q.data_ptr() % 16:
        return "q view not 16-byte aligned"
    return None


def paged_prefill_attention(q: Tensor, k_cache: Tensor, v_cache: Tensor, block_table: Tensor, block_size: int,
                            chunk_start: Tensor, chunk_len: Tensor, chunk_pos: Tensor, scale: float,
                            max_keys: Optional[int] = None) -> Tensor:
    """Causal prefill of query chunks against a paged bf16 cache (prefix caching).  q: [T, h, D], or the grouped view
    [T, h_kv, group, D] (query head kv * group + g); k/v_cache: [slots, h_kv, D] bf16; block_table: int32
    [>= N, max_blocks]; chunk_start / chunk_len / chunk_pos: int32 [N].  Chunk c is queries [chunk_start[c],
    chunk_start[c] + chunk_len[c]); query i of it sits at position chunk_pos[c] + i of the sequence whose table row is
    c and attends to that sequence's keys j <= chunk_pos[c] + i, key j at row block_table[c, j // block_size] *
    block_size + j % block_size.  Returns o [T, h, D]; rows of q outside every chunk are left undefined.
    `max_keys` bounds chunk_pos + chunk_len (the table must cover it); None reads it from the descriptors.  Table
    entries are trusted by the kernel; the reference raises ValueError for one outside the cache's blocks."""
    if isinstance(k_cache, Fp8KV) or isinstance(v_cache, Fp8KV):
        raise TypeError("paged_prefill_attention: fp8 caches are not supported")
    if max_keys is None:
        max_keys = int((chunk_pos.long() + chunk_len.long()).max()) if chunk_len.numel() else 0
    bs = int(block_size)
    if C := _kernels("paged_prefill_attention", q, k_cache, v_cache,
                     unsupported=lambda: _paged_prefill_unsupported(q, bs)):
        return C.paged_prefill_attention(q, k_cache, v_cache, block_table, bs, chunk_start, chunk_len, chunk_pos,
                                         scale, int(max_keys))
    if bs < 1 or bs > 1024 or bs & (bs - 1):
        raise ValueError(f"paged_prefill_attention: block size {bs} is not a power of two up to 1024")
    T, D = q.shape[0], q.shape[-1]
    qf = q.reshape(T, -1, D).float()
    h, h_kv = qf.shape[1], k_cache.shape[1]
    G = h // h_kv
    nblk = (k_cache.shape[0] - 1) // bs
    o = torch.zeros(T, h, D, dtype=q.dtype, device=q.device)
    for c, (s0, n, p0) in enumerate(zip(chunk_start.tolist(), chunk_len.tolist(), chunk_pos.tolist())):
        if n == 0:
            continue
        keys = p0 + n
        if keys > max_keys or keys > block_table.shape[1] * bs:
            raise ValueError(f"paged_prefill_attention: chunk {c} reads {keys} keys, more than max_keys {max_keys} "
                             f"or the {block_table.shape[1]} blocks of a table row")
        j = torch.arange(keys, device=q.device)
        blk = block_table[c].long()[j // bs]
        if bool(((blk < 0) | (blk >= nblk)).any()):
            raise ValueError(f"paged_prefill_attention: chunk {c} reads a block outside the cache's {nblk} blocks")
        rows = blk * bs + j % bs
        k = k_cache[rows].float().repeat_interleave(G, dim=1)                                    # [keys, h, D]
        v = v_cache[rows].float().repeat_interleave(G, dim=1)
        s = torch.einsum("ihd,jhd->hij", qf[s0:s0 + n] * scale, k)
        qpos = p0 + torch.arange(n, device=q.device)
        s = s.masked_fill(j[None, None, :] > qpos[None, :, None], float("-inf"))
        p = torch.softmax(s, dim=-1)
        o[s0:s0 + n] = torch.einsum("hij,jhd->ihd", p, v).to(q.dtype)
    return o


# =================================================================================================
# multi-LoRA segments (serving many adapters over one base model)
# =================================================================================================
LORA_MAX_RANK = 192         # R of the kernels: up to three stacked projections of rank 64


def _lora_unsupported(rows_mat: Tensor, w: Tensor, R: int, inner: int) -> Optional[str]:
    """Why the LoRA kernels cannot take these operands, or None.  rows_mat: x (shrink) or out (expand), w: A or B
    with rank R and other dimension `inner` (K of A, N of B)."""
    if R % 8 or R > LORA_MAX_RANK or inner % 8:
        return "LoRA rank not a multiple of 8 up to 192, or K / N not a multiple of 8"
    if rows_mat.dim() != 2 or rows_mat.stride(-1) != 1 or rows_mat.stride(0) % 8 or rows_mat.data_ptr() % 16:
        return "LoRA rows not 16-byte aligned"
    if not w.is_contiguous() or w.data_ptr() % 16:
        return "LoRA adapters not contiguous"
    return None


def _lora_segments(rows: Tensor, seg_start: Tensor, seg_slot: Tensor):
    starts = seg_start.tolist()
    for s, slot in enumerate(seg_slot.tolist()):
        yield slot, starts[s], starts[s + 1], rows[starts[s]:starts[s + 1]].long()


@torch.library.custom_op("alpa_b200::lora_shrink", mutates_args=())
def lora_shrink(x: Tensor, A: Tensor, rows: Tensor, seg_start: Tensor, seg_slot: Tensor) -> Tensor:
    """LoRA shrink over segments of a token batch.  x: [T, K]; A: [slots, R, K]; rows int32 [Tl] (batch rows grouped
    by segment), seg_start int32 [S + 1], seg_slot int32 [S]: segment s is rows[seg_start[s]:seg_start[s + 1]] and uses
    adapter A[seg_slot[s]].  Returns fp32 partials y [P, Tl, R] whose sum over P is x[rows[i]] . A[slot]^T (the kernel
    splits K into P parts, the reference returns P = 1); `lora_expand_` takes them as they are.  Rows of y outside
    every segment are undefined."""
    if C := _kernels("lora_shrink", x, A, unsupported=lambda: _lora_unsupported(x, A, A.shape[1], A.shape[2])):
        return C.lora_shrink(x, A, rows, seg_start, seg_slot)
    y = torch.zeros(1, rows.shape[0], A.shape[1], dtype=torch.float32, device=x.device)
    for slot, b, e, r in _lora_segments(rows, seg_start, seg_slot):
        y[0, b:e] = x[r].float() @ A[slot].float().T
    return y


@lora_shrink.register_fake
def _(x, A, rows, seg_start, seg_slot):
    return x.new_empty(1, rows.shape[0], A.shape[1], dtype=torch.float32)


@torch.library.custom_op("alpa_b200::lora_expand_", mutates_args=("out",))
def lora_expand_(out: Tensor, y: Tensor, B: Tensor, scale: Tensor, rows: Tensor, seg_start: Tensor,
                 seg_slot: Tensor) -> None:
    """LoRA expand, in place: out[rows[i]] = out[rows[i]] + scale[slot] * (y[:, i].sum(0) . B[slot]^T), rounded once
    to out's dtype.  out: [T, N]; y: [P, Tl, R] fp32 (`lora_shrink`); B: [slots, N, R]; scale: fp32 [slots]
    (lora_alpha / r).  A row of out that no segment lists is neither read nor written."""
    if C := _kernels("lora_expand_", out, B, unsupported=lambda: _lora_unsupported(out, B, B.shape[2], B.shape[1])):
        C.lora_expand_(out, y, B, scale, rows, seg_start, seg_slot)
        return
    ys = y.sum(0)
    for slot, b, e, r in _lora_segments(rows, seg_start, seg_slot):
        out[r] = (out[r].float() + scale[slot].float() * (ys[b:e] @ B[slot].float().T)).to(out.dtype)


# =================================================================================================
# sharding-invariant dropout (counter-based Philox4x32-10 keyed by seed / stream / GLOBAL element index)
# =================================================================================================
_PHILOX_M0, _PHILOX_M1, _PHILOX_W0, _PHILOX_W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_U32 = 0xFFFFFFFF


def _philox4x32_10(c0: Tensor, c1: Tensor, c2: Tensor, c3: Tensor, k0: Tensor, k1: Tensor):
    """Philox4x32-10 on int64 tensors holding 32-bit words (bit-exact with the CUDA kernel)."""
    for _ in range(10):
        p0, p1 = c0 * _PHILOX_M0, c2 * _PHILOX_M1           # wraps mod 2^64: the low 64 bits are exact
        hi0, lo0 = (p0 >> 32) & _U32, p0 & _U32
        hi1, lo1 = (p1 >> 32) & _U32, p1 & _U32
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + _PHILOX_W0) & _U32, (k1 + _PHILOX_W1) & _U32
    return c0, c1, c2, c3


def dropout_keep_mask(local_shape, p: float, seed: Tensor, stream: int, global_shape, offsets, device=None) -> Tensor:
    """Boolean keep-mask of the shard `offsets .. offsets + local_shape` of a tensor of `global_shape`."""
    device = device if device is not None else seed.device
    g = torch.zeros(tuple(local_shape), dtype=torch.int64, device=device)
    stride = 1
    for d in range(len(local_shape) - 1, -1, -1):
        idx = (torch.arange(local_shape[d], device=device, dtype=torch.int64) + int(offsets[d])) * stride
        g = g + idx.view([-1 if i == d else 1 for i in range(len(local_shape))])
        stride *= int(global_shape[d])
    ctr = g >> 2
    sd = seed.to(device=device, dtype=torch.int64).reshape(())
    k0, k1 = sd & _U32, (sd >> 32) & _U32
    words = _philox4x32_10(ctr & _U32, (ctr >> 32) & _U32, torch.full_like(ctr, int(stream) & _U32), torch.zeros_like(ctr),
                           k0.expand_as(ctr), k1.expand_as(ctr))
    lane = g & 3
    r = torch.where(lane == 0, words[0], torch.where(lane == 1, words[1], torch.where(lane == 2, words[2], words[3])))
    threshold = min(4294967295, int(math.floor(p * 4294967296.0)))
    return r >= threshold


@torch.library.custom_op("alpa_b200::dropout", mutates_args=())
def dropout(x: Tensor, p: float, seed: Tensor, stream: int, global_shape: List[int], offsets: List[int]) -> Tensor:
    """y = x / (1 - p) where the element's random word (Philox of seed, stream and its GLOBAL linear index inside a
    tensor of `global_shape`; this shard starts at `offsets`) is >= p * 2^32, else 0.  `seed`: int64 scalar tensor
    (e.g. derived from the step counter).  The mask does not depend on the sharding, so parallel plans reproduce the
    single-device run bit for bit, and the backward pass / a rematerialised forward regenerate it.
    (reference: stateful XLA RNG with per-device seeds, alpa/monkey_patch.py:52-160)"""
    if p <= 0.0:
        return x.clone()
    if C := _kernels("dropout", x, dtypes=(torch.bfloat16, torch.float32),
                     unsupported=None if 1 <= x.dim() <= 6 else "rank outside 1..6"):
        return C.dropout(x, float(p), seed.to(x.device), int(stream), list(global_shape), list(offsets))
    keep = dropout_keep_mask(tuple(x.shape), p, seed, stream, global_shape, offsets, device=x.device)
    return torch.where(keep, x.float() * (1.0 / (1.0 - p)), torch.zeros((), device=x.device)).to(x.dtype)


@dropout.register_fake
def _(x, p, seed, stream, global_shape, offsets):
    return torch.empty_like(x)


def _dropout_setup(ctx, inputs, output):
    _, ctx.p, seed, ctx.stream, ctx.global_shape, ctx.offsets = inputs
    ctx.save_for_backward(seed)


def _dropout_bwd(ctx, dy):
    (seed,) = ctx.saved_tensors
    return dropout(dy, ctx.p, seed, ctx.stream, ctx.global_shape, ctx.offsets), None, None, None, None, None


dropout.register_autograd(_dropout_bwd, setup_context=_dropout_setup)


def dropout_like(x: Tensor, p: float, seed: Tensor, stream: int = 0, training: bool = True) -> Tensor:
    """Convenience wrapper used by the models: whole-tensor dropout (global shape = x.shape)."""
    if not training or p <= 0.0:
        return x
    return dropout(x, p, seed, stream, list(x.shape), [0] * x.dim())


# =================================================================================================
# fp8 weight linear (serving): w is e4m3 with one fp32 scale per output channel
# =================================================================================================
class RMSNormArgs(NamedTuple):
    """The RMSNorm a serving projection applies to its input, y = x * rsqrt(mean(x^2) + eps) * gamma: passed as `ln`
    where a LayerNorm is passed as (gamma, beta, eps)."""
    gamma: Tensor
    eps: float


def norm_rows(x: Tensor, ln: Union[Tuple[Tensor, Tensor, float], RMSNormArgs]) -> Tensor:
    """x normalised by `ln`: a LayerNorm (gamma, beta, eps) or an RMSNormArgs.  Not differentiable: like every `fast`
    entry point it calls the implementations directly, not through the dispatcher."""
    if isinstance(ln, RMSNormArgs):
        return rms_norm._init_fn(x, ln.gamma, ln.eps)[0]
    return layer_norm._init_fn(x, ln[0], ln[1], ln[2])[0]


def linear_decode(x: Tensor, w: Tensor, w_scale: Optional[Tensor], b: Optional[Tensor] = None, act: str = "none",
                  residual: Optional[Tensor] = None,
                  ln: Optional[Union[Tuple[Tensor, Tensor, float], RMSNormArgs]] = None) -> Tensor:
    """y = act(LN(x) @ W^T * w_scale + b) (+ residual) for a handful of tokens (decode): weight-streaming GEMV on
    sm_90a (the streamed fp8 / bf16 weight bytes go to the tensor cores unconverted; with fp8 weights the activations
    are quantised per token to e4m3 inside the kernel, like the prefill fp8 GEMM; no tile padding); not
    differentiable.  x: [..., K] with at most 8 rows in total.  `ln` = (gamma, beta, eps) layer-normalises x inside the
    kernel's prologue (one launch less per projection), `ln` = RMSNormArgs(gamma, eps) RMS-normalises it there; None =
    x is used as is."""
    rows = x.numel() // x.shape[-1]
    K = x.shape[-1]
    fp8w = w.dtype == torch.float8_e4m3fn
    unsupported = ("more than 8 rows" if rows > 8 else
                   "K not a multiple of the GEMV's K step" if K % (64 if fp8w else 32) else
                   "staged activations over 200 KiB" if rows * K * (1 if fp8w else 2) > 200 * 1024 else None)
    if C := _kernels("linear_decode", x, unsupported=unsupported):          # the binding checks w: bf16 or e4m3
        x2 = _as2d(x)
        if x2.stride(0) % 8 or x2.data_ptr() % 16:     # the prologue reads rows 16 bytes at a time
            x2 = x2.contiguous()
        r2 = None if residual is None else _as2d(residual)
        if ln is not None and ln[0].dtype != torch.bfloat16:
            x2 = norm_rows(x2, ln)          # the fused prologue reads bf16 gamma (/ beta)
            ln = None
        if ln is None:
            y = C.gemv_decode(x2, w, w_scale, b, r2, _ACT_IDS[act])
        elif isinstance(ln, RMSNormArgs):
            y = C.gemv_decode(x2, w, w_scale, b, r2, _ACT_IDS[act], ln.gamma, None, float(ln.eps), True)
        else:
            y = C.gemv_decode(x2, w, w_scale, b, r2, _ACT_IDS[act], ln[0], ln[1], float(ln[2]))
        return y.view(*x.shape[:-1], w.shape[0])
    if isinstance(ln, RMSNormArgs):
        x = _rms_ref(x, ln.gamma, ln.eps)[0]
    elif ln is not None:
        x = F.layer_norm(x.float(), (K,), ln[0].float(), ln[1].float(), ln[2]).to(x.dtype)
    wf = w.to(torch.float32) * w_scale[:, None] if w_scale is not None else w.to(torch.float32)
    y = _act_fn(F.linear(x.float(), wf, None if b is None else b.float()), act)
    if residual is not None:
        y = y + residual.float()
    return y.to(x.dtype)


def linear_fp8(x: Tensor, w_fp8: Tensor, w_scale: Tensor, b: Optional[Tensor] = None, act: str = "none") -> Tensor:
    """y = act(x @ (w_fp8 * w_scale[:, None])^T + b).  On sm_90a the activations are quantised per token to e4m3
    and the product runs on the fp8 tensor cores (`kind::f8f6f4`), scales applied in the epilogue; elsewhere the
    weights are dequantised (same maths up to the activation rounding)."""
    if C := _kernels("linear_fp8", x, unsupported=None if x.shape[-1] % 16 == 0 and w_fp8.shape[0] % 8 == 0
                     else "K % 16 or N % 8"):
        x2 = _as2d(x)
        if x2.stride(0) % 8 or x2.data_ptr() % 16:     # the quantiser reads rows 16 bytes at a time
            x2 = x2.contiguous()
        return C.gemm_fp8(x2, w_fp8, w_scale, b, _ACT_IDS[act]).view(*x.shape[:-1], w_fp8.shape[0])
    w = (w_fp8.to(torch.float32) * w_scale[:, None]).to(x.dtype)
    y = F.linear(x, w, b)
    return _act_fn(y, act)


# =================================================================================================
# cross-mesh resharding pack / unpack: the tiles one device exchanges with a peer as ONE contiguous message
# =================================================================================================
def packed_nbytes(views: List[Tensor]) -> int:
    """Bytes of the staging buffer of `views` (every tile starts on a 16-byte boundary)."""
    return sum((v.numel() * v.element_size() + 15) // 16 * 16 for v in views)


def _tiles_unsupported(views: List[Tensor]) -> Optional[str]:
    """Why the pack kernel cannot move these tiles (non-empty, 1-D to 4-D, rows contiguous), or None."""
    ok = all(1 <= v.dim() <= 4 and v.stride(-1) == 1 and v.numel() > 0 for v in views)
    return None if ok else "tile empty, over 4-D or with strided rows"


def pack_tiles(views: List[Tensor], flat: Optional[Tensor] = None) -> Tensor:
    """Gather strided slices into one uint8 staging buffer (one launch on sm_90a: pack_sm90.cu)."""
    if flat is None:
        flat = torch.empty(packed_nbytes(views), dtype=torch.uint8, device=views[0].device)
    C = _kernels("pack_tiles", flat, *views, dtypes=None,
                 unsupported=lambda: _tiles_unsupported(views)) if views else None
    if C is not None:
        C.pack_tiles(list(views), flat, False)
        return flat
    off = 0
    for v in views:
        n = v.numel() * v.element_size()
        flat[off:off + n].copy_(v.contiguous().view(-1).view(torch.uint8))
        off += (n + 15) // 16 * 16
    return flat


def unpack_tiles(flat: Tensor, views: List[Tensor]) -> None:
    """Scatter a received staging buffer into the destination slices (in place)."""
    C = _kernels("unpack_tiles", flat, *views, dtypes=None,
                 unsupported=lambda: _tiles_unsupported(views)) if views else None
    if C is not None:
        C.pack_tiles(list(views), flat, True)
        return
    off = 0
    for v in views:
        n = v.numel() * v.element_size()
        v.copy_(flat[off:off + n].view(v.dtype).view(v.shape))
        off += (n + 15) // 16 * 16


# =================================================================================================
# block-scaled MXFP8 (OCP microscaling): e4m3 elements + one UE8M0 scale per 32 K elements; the scales are applied
# inside the tensor core (one wgmma per 32-element block with the scales folded in registers, gemm_sm90.cu).  Scale factors are stored in
# the atom layout the instruction reads: [ceil(rows/128), ceil(K/128), 512] bytes, byte (r, j) of an atom at
# (r % 32) * 16 + (r // 32) * 4 + j  (r = row inside the 128-row group, j = K block inside the 128-element slice).
# =================================================================================================
MX_BLOCK = 32


def _mx_exponents(amax: Tensor) -> Tensor:
    """Smallest e (clamped to [-127, 127]) with amax / 2^e <= 448 (the e4m3 maximum); -127 for all-zero blocks."""
    a = amax.double()
    e = torch.ceil(torch.log2(torch.clamp(a, min=1e-300) / 448.0))
    e = torch.where(a * torch.exp2(-e) > 448.0, e + 1, e)                  # log2 rounding: verify, then tighten
    e = torch.where(a * torch.exp2(-(e - 1)) <= 448.0, e - 1, e)
    e = torch.where(a > 0, e, torch.full_like(e, -127.0))
    return e.clamp(-127, 127).to(torch.int32)


def mx_pack_scale_atoms(e: Tensor) -> Tensor:
    """Biased exponents [rows, K/32] (uint8 values) -> scale atoms [ceil(rows/128), ceil(K/128), 512] (padding = 127)."""
    R, KB = e.shape
    RG, KA = (R + 127) // 128, (KB + 3) // 4
    full = torch.full((RG * 128, KA * 4), 127, dtype=torch.uint8, device=e.device)
    full[:R, :KB] = e.to(torch.uint8)
    # [RG, quadrant q = r // 32, r32 = r % 32, KA, j] -> [RG, KA, r32, q, j]
    return full.view(RG, 4, 32, KA, 4).permute(0, 3, 2, 1, 4).reshape(RG, KA, 512).contiguous()


def mx_unpack_scale_atoms(sf: Tensor, rows: int, K: int) -> Tensor:
    """Inverse of `mx_pack_scale_atoms`: atoms -> biased exponents [rows, K/32] (uint8)."""
    RG, KA, _ = sf.shape
    full = sf.view(RG, KA, 32, 4, 4).permute(0, 3, 2, 1, 4).reshape(RG * 128, KA * 4)
    return full[:rows, :K // MX_BLOCK].contiguous()


def _quantize_mxfp8_ref(x: Tensor) -> Tuple[Tensor, Tensor]:
    M, K = x.shape
    xb = x.float().view(M, K // MX_BLOCK, MX_BLOCK)
    e = _mx_exponents(xb.abs().amax(-1))
    q = (xb * torch.exp2(-e.float())[..., None]).clamp(-448.0, 448.0).view(M, K).to(torch.float8_e4m3fn)
    return q, mx_pack_scale_atoms((e + 127).to(torch.uint8))


def quantize_mxfp8(x: Tensor) -> Tuple[Tensor, Tensor]:
    """x [rows, K] (K % 32 == 0) -> (q e4m3 [rows, K], scale atoms uint8 [ceil(rows/128), ceil(K/128), 512])."""
    assert x.dim() == 2 and x.shape[1] % MX_BLOCK == 0, "quantize_mxfp8: [rows, K] with K % 32 == 0"
    if C := _kernels("quantize_mxfp8", x):
        ok = x.stride(-1) == 1 and x.stride(0) % 8 == 0 and x.data_ptr() % 16 == 0
        q, sf = C.quantize_mxfp8(x if ok else x.contiguous())
        return q, sf
    return _quantize_mxfp8_ref(x)


def dequantize_mxfp8(q: Tensor, sf: Tensor) -> Tensor:
    """fp32 values of a block-scaled tensor (the numerics oracle of the kernel)."""
    rows, K = q.shape
    e = mx_unpack_scale_atoms(sf, rows, K).to(torch.float32) - 127.0
    return (q.to(torch.float32).view(rows, K // MX_BLOCK, MX_BLOCK) * torch.exp2(e)[..., None]).view(rows, K)


def linear_mxfp8(x: Tensor, w_q: Tensor, w_sf: Tensor, b: Optional[Tensor] = None, act: str = "none") -> Tensor:
    """y = act(x @ dequant(w_q, w_sf)^T + b) with block-scaled fp8 operands.  On sm_90a the activations are
    block-quantised on the fly and the product runs on `wgmma` e4m3 with the block scales folded in per K = 32 step (scales in
    memory); elsewhere both operands are dequantised -- the same maths, activation rounding included."""
    K, N = x.shape[-1], w_q.shape[0]
    x2 = _as2d(x)
    if C := _kernels("linear_mxfp8", x, unsupported=None if K % MX_BLOCK == 0 and N % 8 == 0 else "K % 32 or N % 8"):
        if x2.stride(0) % 8 or x2.data_ptr() % 16:         # the quantiser reads rows 16 bytes at a time
            x2 = x2.contiguous()
        return C.gemm_mxfp8(x2, w_q, w_sf, b, _ACT_IDS[act]).view(*x.shape[:-1], N)
    xq, x_sf = _quantize_mxfp8_ref(x2)
    y = F.linear(dequantize_mxfp8(xq, x_sf), dequantize_mxfp8(w_q, w_sf), None if b is None else b.float())
    return _act_fn(y, act).to(x.dtype).view(*x.shape[:-1], N)


# =================================================================================================
# batched GEMM (per-expert FFN of the MoE layer) -- same operand convention as the native kernel:
#   a: [B, M, K] (trans_a=False) or [B, K, M];   b: [B, N, K] (trans_b=False) or [B, K, N]
# =================================================================================================
@torch.library.custom_op("alpa_b200::bmm", mutates_args=())
def bmm(a: Tensor, b: Tensor, trans_a: bool, trans_b: bool) -> Tensor:
    """C[B, M, N] = op(a) @ op(b)^T-convention (see above)"""
    if C := _kernels("bmm", a, b, unsupported=lambda: _gemm_unsupported(a, b)):
        return C.gemm(a, b, trans_a, trans_b)
    am = a.transpose(-1, -2) if trans_a else a
    bm = b if trans_b else b.transpose(-1, -2)
    return torch.matmul(am, bm)


@bmm.register_fake
def _(a, b, trans_a, trans_b):
    M = a.shape[-1] if trans_a else a.shape[-2]
    N = b.shape[-1] if trans_b else b.shape[-2]
    return a.new_empty(*a.shape[:-2], M, N)


def _bmm_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)
    a, b, ta, tb = inputs
    ctx.save_for_backward(a, b)
    ctx.flags = (ta, tb)


def _bmm_bwd(ctx, dc):
    if dc is None:
        return None, None, None, None
    a, b = ctx.saved_tensors
    ta, tb = ctx.flags
    da = db = None
    if ctx.needs_input_grad[0]:
        da = bmm(b, dc, not tb, False) if ta else bmm(dc, b, False, not tb)
    if ctx.needs_input_grad[1]:
        db = bmm(a, dc, not ta, True) if tb else bmm(dc, a, True, not ta)
    return da, db, None, None


bmm.register_autograd(_bmm_bwd, setup_context=_bmm_setup)


# =================================================================================================
# MoE token routing: index-based dispatch / combine (GShard top-2).  The reference builds dense one-hot
# [G,S,E,C] masks and einsums (alpa/model/moe.py:144-186); these are the same maps as gathers/scatters.
#   expert, slot: int64 [G, S, K]; slot < 0 = token dropped for that choice
#   dispatched buffer: [E, G*C, M], row g*C + c of expert e
# =================================================================================================
@torch.library.custom_op("alpa_b200::moe_top2_route", mutates_args=())
def moe_top2_route(gates: Tensor, capacity: int) -> Tuple[Tensor, Tensor]:
    """GShard top-2 routing of gate probabilities [G,S,E] (reference: top2_gating, alpa/model/moe.py:85-141)
    -> (expert [G,S,2], slot [G,S,2]) int64.  First choices fill an expert's capacity in token order, second
    choices continue after them; slot = -1 when the expert is full."""
    G, S, E = gates.shape
    C = _kernels("moe_top2_route", gates, dtypes=None)     # the kernel reads the gates as fp32
    if C is not None:
        return tuple(C.moe_top2_route(gates.float().contiguous(), capacity))
    idx1 = gates.argmax(-1)
    mask1 = F.one_hot(idx1, E)
    idx2 = (gates * (1 - mask1)).argmax(-1)
    mask2 = F.one_hot(idx2, E)
    pos1_all = mask1.cumsum(-2) - mask1
    keep1 = (pos1_all < capacity) & mask1.bool()
    pos1 = (pos1_all * keep1).sum(-1)
    ok1 = keep1.any(-1)
    count1 = keep1.sum(-2)
    pos2_all = (mask2.cumsum(-2) - mask2) + count1.unsqueeze(-2)
    keep2 = (pos2_all < capacity) & mask2.bool()
    pos2 = (pos2_all * keep2).sum(-1)
    ok2 = keep2.any(-1)
    expert = torch.stack([idx1, idx2], -1)
    slot = torch.stack([torch.where(ok1, pos1, torch.full_like(pos1, -1)),
                        torch.where(ok2, pos2, torch.full_like(pos2, -1))], -1)
    return expert, slot


@moe_top2_route.register_fake
def _(gates, capacity):
    G, S, _ = gates.shape
    return (gates.new_empty(G, S, 2, dtype=torch.int64), gates.new_empty(G, S, 2, dtype=torch.int64))


@torch.library.custom_op("alpa_b200::moe_dispatch", mutates_args=())
def moe_dispatch(x: Tensor, expert: Tensor, slot: Tensor, weight: Optional[Tensor], num_experts: int,
                 capacity: int) -> Tensor:
    """d[e, g*C+c, :] = (weight[g,s,k] *) x[g,s,:] for every routed (g,s,k); zeros in unused slots"""
    G, S, M = x.shape
    K = expert.shape[-1]
    if C := _kernels("moe_dispatch", x, weight, unsupported=None if M % 8 == 0 else "M not a multiple of 8"):
        d = torch.zeros(num_experts, G * capacity, M, device=x.device, dtype=x.dtype)
        C.moe_dispatch_(x.contiguous(), expert.contiguous(), slot.contiguous(),
                        None if weight is None else weight.contiguous(), d, capacity)
        return d
    d = torch.zeros(num_experts * G * capacity + 1, M, device=x.device, dtype=x.dtype)
    g = torch.arange(G, device=x.device).view(G, 1, 1)
    row = (expert * G + g) * capacity + slot
    row = torch.where(slot >= 0, row, torch.full_like(row, num_experts * G * capacity)).reshape(-1)
    src = x.unsqueeze(2).expand(G, S, K, M)
    if weight is not None:
        src = src * weight.unsqueeze(-1).to(x.dtype)
    d.index_copy_(0, row, src.reshape(-1, M))
    return d[:-1].view(num_experts, G * capacity, M)


@moe_dispatch.register_fake
def _(x, expert, slot, weight, num_experts, capacity):
    return x.new_empty(num_experts, x.shape[0] * capacity, x.shape[2])


@torch.library.custom_op("alpa_b200::moe_combine", mutates_args=())
def moe_combine(eo: Tensor, expert: Tensor, slot: Tensor, weight: Optional[Tensor]) -> Tensor:
    """out[g,s,:] = sum_k weight[g,s,k] * eo[expert[g,s,k], g*C + slot[g,s,k], :]  (weight=None: 1)"""
    E, GC, M = eo.shape
    G, S, K = expert.shape
    cap = GC // G
    if C := _kernels("moe_combine", eo, weight, unsupported=None if M % 8 == 0 else "M not a multiple of 8"):
        return C.moe_combine(eo.contiguous(), expert.contiguous(), slot.contiguous(),
                             None if weight is None else weight.contiguous())
    g = torch.arange(G, device=eo.device).view(G, 1, 1)
    ok = slot >= 0
    row = torch.where(ok, (expert * G + g) * cap + slot, torch.zeros_like(slot))
    rows = eo.reshape(E * GC, M)[row.reshape(-1)].view(G, S, K, M).float()
    w = ok.float() if weight is None else weight.float() * ok.float()
    return (rows * w.unsqueeze(-1)).sum(2).to(eo.dtype)


@moe_combine.register_fake
def _(eo, expert, slot, weight):
    G, S, _ = expert.shape
    return eo.new_empty(G, S, eo.shape[-1])


@torch.library.custom_op("alpa_b200::moe_combine_wgrad", mutates_args=())
def moe_combine_wgrad(dout: Tensor, eo: Tensor, expert: Tensor, slot: Tensor) -> Tensor:
    """dweight[g,s,k] = <dout[g,s,:], eo[expert, g*C+slot, :]> (0 for dropped choices)"""
    E, GC, M = eo.shape
    G, S, K = expert.shape
    cap = GC // G
    if C := _kernels("moe_combine_wgrad", eo, dout, unsupported=None if M % 8 == 0 else "M not a multiple of 8"):
        return C.moe_combine_wgrad(dout.contiguous(), eo.contiguous(), expert.contiguous(), slot.contiguous())
    g = torch.arange(G, device=eo.device).view(G, 1, 1)
    ok = slot >= 0
    row = torch.where(ok, (expert * G + g) * cap + slot, torch.zeros_like(slot))
    rows = eo.reshape(E * GC, M)[row.reshape(-1)].view(G, S, K, M).float()
    dw = (rows * dout.float().unsqueeze(2)).sum(-1) * ok.float()
    return dw.to(dout.dtype)


@moe_combine_wgrad.register_fake
def _(dout, eo, expert, slot):
    return dout.new_empty(*expert.shape)


def _dispatch_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)
    x, expert, slot, weight, E, C = inputs
    ctx.save_for_backward(expert, slot, weight, x if weight is not None else None)
    ctx.has_w = weight is not None


def _dispatch_bwd(ctx, dd):
    if dd is None:
        return None, None, None, None, None, None
    expert, slot, weight, x = ctx.saved_tensors
    dx = moe_combine(dd, expert, slot, weight) if ctx.needs_input_grad[0] else None
    dw = None
    if ctx.has_w and ctx.needs_input_grad[3]:
        dw = moe_combine_wgrad(x, dd, expert, slot)
    return dx, None, None, dw, None, None


moe_dispatch.register_autograd(_dispatch_bwd, setup_context=_dispatch_setup)


def _combine_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)
    eo, expert, slot, weight = inputs
    ctx.save_for_backward(eo, expert, slot, weight)
    ctx.dims = (eo.shape[0], eo.shape[1] // expert.shape[0])


def _combine_bwd(ctx, dout):
    if dout is None:
        return None, None, None, None
    eo, expert, slot, weight = ctx.saved_tensors
    E, C = ctx.dims
    deo = moe_dispatch(dout, expert, slot, weight, E, C) if ctx.needs_input_grad[0] else None
    dw = None
    if weight is not None and ctx.needs_input_grad[3]:
        dw = moe_combine_wgrad(dout, eo, expert, slot)
    return deo, None, None, dw


moe_combine.register_autograd(_combine_bwd, setup_context=_combine_setup)


# =================================================================================================
# softmax cross entropy over the last dim (optionally a vocab shard)
# =================================================================================================
@torch.library.custom_op("alpa_b200::cross_entropy", mutates_args=())
def cross_entropy(logits: Tensor, labels: Tensor, vocab_start: int = 0) -> Tuple[Tensor, Tensor]:
    """Per-token statistics over the local vocab shard: (stats[T,3]=(max, sum exp(x-max), target logit)).
    Returned as (loss[T], stats[T,3]); loss is the full NLL when the shard is the whole vocabulary."""
    T = labels.numel()
    V = logits.shape[-1]
    l2 = logits.reshape(T, V)
    lab = labels.reshape(T)
    aligned = V % 8 == 0 and l2.stride(0) % 8 == 0 and l2.stride(1) == 1
    if C := _kernels("cross_entropy", logits, unsupported=None if aligned else "vocab rows not 16-byte aligned"):
        stats = C.ce_stats(l2, lab.contiguous(), vocab_start)
    else:
        lf = l2.float()
        mx = lf.max(dim=1).values
        se = torch.exp(lf - mx[:, None]).sum(1)
        local = lab - vocab_start
        ok = (local >= 0) & (local < V)
        tgt = lf.gather(1, local.clamp(0, V - 1)[:, None])[:, 0] * ok.float()
        stats = torch.stack([mx, se, tgt], dim=1)
    loss = torch.log(stats[:, 1]) + stats[:, 0] - stats[:, 2]
    return loss.view(labels.shape), stats


@cross_entropy.register_fake
def _(logits, labels, vocab_start=0):
    T = labels.numel()
    return logits.new_empty(labels.shape, dtype=torch.float32), logits.new_empty(T, 3, dtype=torch.float32)


@torch.library.custom_op("alpa_b200::cross_entropy_bwd", mutates_args=())
def cross_entropy_bwd(logits: Tensor, labels: Tensor, stats: Tensor, dloss: Tensor, vocab_start: int = 0) -> Tensor:
    """dlogits = (softmax(logits) - onehot(labels)) * dloss[token]; stats = global (max, sumexp)."""
    T = labels.numel()
    V = logits.shape[-1]
    lab = labels.reshape(T)
    if C := _kernels("cross_entropy_bwd", logits, unsupported=None if V % 8 == 0 else "V not a multiple of 8"):
        g = logits.reshape(T, V).clone()
        C.ce_grad_(g, lab.contiguous(), stats[:, :2].contiguous(), dloss.reshape(T).float().contiguous(), vocab_start)
        return g.view(logits.shape)
    lf = logits.reshape(T, V).float()
    p = torch.exp(lf - stats[:, 0:1]) / stats[:, 1:2]
    local = lab - vocab_start
    ok = (local >= 0) & (local < V)
    onehot = torch.zeros_like(p)
    onehot.scatter_(1, local.clamp(0, V - 1)[:, None], ok.float()[:, None])
    g = (p - onehot) * dloss.reshape(T, 1).float()
    return g.to(logits.dtype).view(logits.shape)


@cross_entropy_bwd.register_fake
def _(logits, labels, stats, dloss, vocab_start=0):
    return torch.empty_like(logits)


def _ce_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)  # unused outputs yield None, not a zero tensor + add
    logits, labels, vocab_start = inputs
    _, stats = output
    ctx.save_for_backward(logits, labels, stats)
    ctx.vocab_start = vocab_start


def _ce_bwd(ctx, dloss, dstats):
    if dloss is None:
        return None, None, None
    logits, labels, stats = ctx.saved_tensors
    return cross_entropy_bwd(logits, labels, stats, dloss, ctx.vocab_start), None, None


cross_entropy.register_autograd(_ce_bwd, setup_context=_ce_setup)


# =================================================================================================
# fused multi-tensor AdamW (in place): fp32 master/m/v, optional bf16 model copy
# =================================================================================================
_adam_table_cache = {}


@torch.library.custom_op("alpa_b200::fused_adamw_", mutates_args=("masters", "ms", "vs", "params"))
def fused_adamw_(params: List[Tensor], masters: List[Tensor], ms: List[Tensor], vs: List[Tensor],
                 grads: List[Tensor], step: Tensor, lr: float, beta1: float, beta2: float, eps: float,
                 weight_decays: List[float], grad_scale: float) -> None:
    """`step` is the 1-based step count as a scalar tensor (read on the device by the kernel).
    One launch updates every parameter: master -= lr * (m_hat / (sqrt(v_hat)+eps) + wd * master);
    params (bf16 compute copies, may alias masters when training in fp32) are refreshed in the same pass."""
    if C := _kernels("fused_adamw_", *masters, *grads, dtypes=(torch.float32, torch.bfloat16)):
        # Non-contiguous gradients are copied into persistent contiguous staging buffers every step (the
        # device table points at the staging buffer, which the cache entry keeps alive).
        key = tuple((t.data_ptr(), t.numel(), t.dtype, t.is_contiguous())
                    for t in (*grads, *masters, *ms, *vs, *params)) + tuple(weight_decays)
        ent = _adam_table_cache.get(key)
        if ent is None:
            pb = [p if (p.dtype == torch.bfloat16 and p.data_ptr() != m.data_ptr()) else None
                  for p, m in zip(params, masters)]
            staging = [None if g.is_contiguous() else torch.empty(g.shape, dtype=g.dtype, device=g.device)
                       for g in grads]
            gsrc = [g if st is None else st for g, st in zip(grads, staging)]
            tab = C.adam_build_tables(gsrc, masters, ms, vs, pb, list(weight_decays))
            if len(_adam_table_cache) > 64:
                _adam_table_cache.clear()
            # the entry owns the staging buffers and the optimizer state the table points at; gradients are looked
            # up by (address, numel, dtype), so a recycled address holding an identically shaped gradient is the
            # same table and anything else is a different key (holding the gradients themselves would pin them)
            ent = (tab, staging, (list(masters), list(ms), list(vs), list(params)))
            _adam_table_cache[key] = ent
        tab, staging = ent[0], ent[1]
        for g, st in zip(grads, staging):
            if st is not None:
                st.copy_(g)
        C.adamw_step(tab[0], tab[1], lr, beta1, beta2, eps, 1, grad_scale, None, step.float().reshape(1))
        return
    stepf = float(step)
    bc1 = 1.0 - beta1 ** stepf
    bc2 = 1.0 - beta2 ** stepf
    for p, w, m, v, g, wd in zip(params, masters, ms, vs, grads, weight_decays):
        gf = g.float() * grad_scale
        m.mul_(beta1).add_(gf, alpha=1 - beta1)
        v.mul_(beta2).addcmul_(gf, gf, value=1 - beta2)
        upd = (m / bc1) / ((v / bc2).sqrt() + eps) + wd * w
        w.add_(upd, alpha=-lr)
        if p.data_ptr() != w.data_ptr():
            p.copy_(w)


@fused_adamw_.register_fake
def _(params, masters, ms, vs, grads, step, lr, beta1, beta2, eps, weight_decays, grad_scale):
    return None


# =================================================================================================
# pipeline / gradient markers (identity on data; reference: alpa/pipeline_parallel/primitive_def.py)
# =================================================================================================
@torch.library.custom_op("alpa_b200::pipeline_marker", mutates_args=())
def pipeline_marker(xs: List[Tensor], name: str, mark_type: str) -> List[Tensor]:
    """Identity marker. mark_type in {"start", "end", "boundary", "grad", "hook"}."""
    return [x.clone() for x in xs]


@pipeline_marker.register_fake
def _(xs, name, mark_type):
    return [torch.empty_like(x) for x in xs]


def _marker_setup(ctx, inputs, output):
    xs, name, mark_type = inputs
    ctx.name, ctx.mark_type = name, mark_type
    ctx.n = len(xs)


def _marker_bwd(ctx, *douts):
    # backward of a boundary is a boundary of the backward pass (same layer name)
    grads = douts[0] if (len(douts) == 1 and isinstance(douts[0], (list, tuple))) else list(douts)
    mt = {"start": "end", "end": "start"}.get(ctx.mark_type, ctx.mark_type)
    outs = pipeline_marker([g for g in grads], ctx.name + "@bwd", mt)
    return outs, None, None


pipeline_marker.register_autograd(_marker_bwd, setup_context=_marker_setup)


# =================================================================================================
# direct entry points
# =================================================================================================
# Calling a `torch.library.custom_op` goes through the PyTorch dispatcher and the custom-op Python trampoline
# (tens to hundreds of microseconds per call); the traced graph needs that, an executor replaying an already planned
# program does not.  `DIRECT_IMPL` maps every alpa_b200 OpOverload to its plain Python implementation (which launches
# the sm_90a kernel), `fast` exposes the same functions by name for inference code that never differentiates.
def _collect_direct():
    from torch._library.custom_ops import CustomOpDef
    table, ns = {}, {}
    for name, obj in list(globals().items()):
        if isinstance(obj, CustomOpDef):
            table[obj._opoverload] = obj._init_fn
            ns[name] = obj._init_fn
    return table, ns


DIRECT_IMPL, _fast_ns = _collect_direct()


def _linear_wgrad_out(dy: Tensor, x: Tensor, out: Tensor) -> Tensor:
    """linear_wgrad writing dw straight into `out` (a slice of a gradient bucket): no pack copy before the collective."""
    v = cache(lambda: (_as2d(dy), _as2d(x)))
    # an `out` the epilogue cannot store to directly is no fallback: linear_wgrad runs and its result is copied
    out_ok = out.dtype == torch.bfloat16 and out.stride(-1) == 1 and out.data_ptr() % 16 == 0 and out.stride(0) % 8 == 0
    if out_ok and (C := _kernels("linear_wgrad", dy, x, unsupported=lambda: _gemm_unsupported(*v()))):
        C.gemm(*v(), True, True, out=out)
        return out
    out.copy_(linear_wgrad._init_fn(dy, x))
    return out


# ops that can produce their result directly in a caller-provided buffer (executor: gradient buckets)
DIRECT_OUT_IMPL = {linear_wgrad._opoverload: _linear_wgrad_out}


def _attention_cached_inplace(q, k_new, v_new, k_cache, v_cache, cache_len, scale):
    return attention_cached_(q, k_new, v_new, k_cache, v_cache, cache_len, scale), k_cache, v_cache


# ops with an in-place form the executor may use when the operands at the listed positions are donated buffers that
# die at this op: overload -> (callable with the same signature and results, operand positions updated in place)
INPLACE_IMPL = {attention_cached._opoverload: (_attention_cached_inplace, (3, 4))}


class _FastNamespace:
    def __init__(self, fns):
        self.__dict__.update(fns)
        self.linear_fp8 = linear_fp8
        self.linear_decode = linear_decode
        self.decode_attention = decode_attention
        self.decode_attention_gqa = decode_attention_gqa
        self.norm_rows = norm_rows
        self.ragged_attention = ragged_attention
        self.paged_prefill_attention = paged_prefill_attention
        self.linear_mxfp8 = linear_mxfp8
        self.Fp8KV = Fp8KV
        self.kv_cache_store = kv_cache_store
        self.kv_cache_load = kv_cache_load


fast = _FastNamespace(_fast_ns)
__all__ += ["DIRECT_IMPL", "DIRECT_OUT_IMPL", "INPLACE_IMPL", "fast"]
