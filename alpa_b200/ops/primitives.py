"""Primitive operators (torch.library custom ops, namespace ``alpa_b200``).

See ``alpa_b200/ops/__init__.py`` for the contract.  The reference has no counterpart file: its
primitives are XLA HLO ops lowered to cuBLAS / LLVM fusions (SURVEY.md §2.5 K1-K9); here they are the
hand-written sm_90a kernels, and the *same* op names appear in traced graphs, plans and programs.
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor

from alpa_b200.global_env import global_config

__all__ = [
    "linear", "linear_act", "linear_dgrad", "linear_dgrad_add", "linear_wgrad", "bias_grad", "act_bwd", "layer_norm",
    "add_layer_norm", "layer_norm_bwd", "attention", "attention_bwd", "attention_qkvpacked",
    "attention_qkvpacked_bwd", "embedding", "embedding_bwd",
    "cross_entropy", "cross_entropy_bwd", "fused_adamw_", "pipeline_marker", "uses_native",
    "bmm", "moe_dispatch", "moe_combine", "moe_combine_wgrad", "moe_top2_route", "linear_fp8", "linear_decode", "attention_decode", "decode_attention", "ragged_attention",
    "attention_cached", "attention_cached_", "quantize_mxfp8", "dequantize_mxfp8", "linear_mxfp8", "mx_pack_scale_atoms",
    "mx_unpack_scale_atoms", "pack_tiles", "unpack_tiles", "packed_nbytes",
    "dropout", "dropout_like", "dropout_keep_mask",
]

_ACT_IDS = {"none": 0, "gelu": 1, "relu": 2}
_DACT_IDS = {"gelu": 3, "relu": 4}


def _native():
    from alpa_b200 import ops
    return ops.native_module()


def uses_native(*tensors: Tensor) -> bool:
    """True if the sm_90a kernels serve this call: CUDA + bf16 activations.  On CUDA/bf16 a missing
    extension is an error (no silent eager fallback) unless ALPA_B200_ALLOW_FALLBACK=1."""
    ts = [t for t in tensors if t is not None]
    if not ts or not all(t.is_cuda for t in ts):
        return False
    if not global_config.use_native_kernels:
        return False
    if not all(t.dtype == torch.bfloat16 for t in ts if t.is_floating_point()):
        return False
    from alpa_b200 import ops
    if ops.native_available():
        return True
    if ops.allow_fallback():
        return False
    raise RuntimeError("alpa_b200: CUDA bf16 tensors but the sm_90a extension is not built/loaded "
                       "(run `python -m alpa_b200.ops.build`; set ALPA_B200_ALLOW_FALLBACK=1 to use PyTorch)")


_FALLBACK_SEEN = set()


def library_fallbacks():
    """Operand layouts for which a primitive fell back to a PyTorch library kernel although the sm_90a extension is
    loaded (shape / stride / alignment outside the wgmma kernel's TMA constraints).  One warning per distinct
    layout is logged; tests and benchmarks can assert this stays empty."""
    return sorted(_FALLBACK_SEEN)


def _gemm_ok(*mats: Tensor) -> bool:
    for m in mats:
        bad = None
        if m.dim() not in (2, 3) or m.stride(-1) != 1 or m.shape[-1] % 8 or m.shape[-2] % 8:
            bad = "shape"
        elif m.stride(-2) % 8 or m.data_ptr() % 16:
            bad = "alignment"
        if bad is not None:
            key = (bad, tuple(m.shape), tuple(m.stride()))
            if key not in _FALLBACK_SEEN:
                _FALLBACK_SEEN.add(key)
                import logging
                logging.getLogger(__name__).warning(
                    "alpa_b200: GEMM operand %s (strides %s) is outside the sm_90a kernel's TMA constraints (%s): "
                    "this call uses the PyTorch library kernel", tuple(m.shape), tuple(m.stride()), bad)
            return False
    return True


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
    if uses_native(x, w, b):
        x2 = _as2d(x)
        if _gemm_ok(x2, w):
            y = _native().gemm(x2, w, False, False, bias=b)
            return y.view(*x.shape[:-1], w.shape[0])
    return F.linear(x, w, b)


@linear.register_fake
def _(x, w, b=None):
    return x.new_empty(*x.shape[:-1], w.shape[0])


@torch.library.custom_op("alpa_b200::linear_act", mutates_args=())
def linear_act(x: Tensor, w: Tensor, b: Optional[Tensor], act: str) -> Tuple[Tensor, Tensor]:
    """(act(z), z) with z = x @ w^T + b; the pre-activation z is kept for the backward pass."""
    if uses_native(x, w, b):
        x2 = _as2d(x)
        if _gemm_ok(x2, w):
            z = torch.empty(x2.shape[0], w.shape[0], device=x.device, dtype=x.dtype)
            y = _native().gemm(x2, w, False, False, bias=b, aux_out=z, act=_ACT_IDS[act])
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
    if uses_native(dy, w):
        d2 = _as2d(dy)
        if _gemm_ok(d2, w):
            dx = _native().gemm(d2, w, False, True)
            return dx.view(*dy.shape[:-1], w.shape[1])
    return torch.matmul(dy, w)


@linear_dgrad.register_fake
def _(dy, w):
    return dy.new_empty(*dy.shape[:-1], w.shape[1])


@torch.library.custom_op("alpa_b200::linear_dgrad_act", mutates_args=())
def linear_dgrad_act(dy: Tensor, w: Tensor, z: Tensor, act: str) -> Tensor:
    """dz = (dy @ w) * act'(z): the activation backward fused into the dgrad epilogue."""
    if uses_native(dy, w, z):
        d2, z2 = _as2d(dy), _as2d(z)
        if _gemm_ok(d2, w) and z2.is_contiguous():
            dx = _native().gemm(d2, w, False, True, aux_in=z2, act=_DACT_IDS[act])
            return dx.view(*dy.shape[:-1], w.shape[1])
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
    if uses_native(dy, w, r):
        d2, r2 = _as2d(dy), _as2d(r)
        if _gemm_ok(d2, w) and r2.is_contiguous() and r2.shape == (d2.shape[0], w.shape[1]):
            dx = _native().gemm(d2, w, False, True, residual=r2)
            return dx.view(*dy.shape[:-1], w.shape[1])
    return torch.matmul(dy, w) + r


@linear_dgrad_add.register_fake
def _(dy, w, r):
    return dy.new_empty(*dy.shape[:-1], w.shape[1])


@torch.library.custom_op("alpa_b200::linear_wgrad", mutates_args=())
def linear_wgrad(dy: Tensor, x: Tensor) -> Tensor:
    """dw[N, K] = dy[..., N]^T @ x[..., K]"""
    if uses_native(dy, x):
        d2, x2 = _as2d(dy), _as2d(x)
        if _gemm_ok(d2, x2):
            return _native().gemm(d2, x2, True, True)
    d2 = dy.reshape(-1, dy.shape[-1])
    x2 = x.reshape(-1, x.shape[-1])
    return torch.matmul(d2.t(), x2)


@linear_wgrad.register_fake
def _(dy, x):
    return dy.new_empty(dy.shape[-1], x.shape[-1])


@torch.library.custom_op("alpa_b200::bias_grad", mutates_args=())
def bias_grad(dy: Tensor) -> Tensor:
    """db[N] = sum over all leading dims of dy[..., N]"""
    if uses_native(dy):
        d2 = _as2d(dy)
        if d2.shape[1] % 8 == 0 and d2.stride(0) % 8 == 0 and d2.data_ptr() % 16 == 0:
            out = torch.zeros(d2.shape[1], device=dy.device, dtype=torch.float32)
            _native().colsum_(d2, out)
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


@torch.library.custom_op("alpa_b200::layer_norm", mutates_args=())
def layer_norm(x: Tensor, g: Tensor, b: Tensor, eps: float) -> Tuple[Tensor, Tensor, Tensor]:
    """(y, mean, rstd); statistics are fp32 with shape x.shape[:-1]."""
    if uses_native(x, g, b) and x.shape[-1] % 8 == 0 and x.shape[-1] <= 8192:
        y, mean, rstd, _ = _native().layernorm_fwd(x.contiguous(), None, g, b, eps, False)
        return y, mean.view(x.shape[:-1]), rstd.view(x.shape[:-1])
    return _ln_ref(x, g, b, eps)


@layer_norm.register_fake
def _(x, g, b, eps):
    st = x.new_empty(x.shape[:-1], dtype=torch.float32)
    return torch.empty_like(x), st, torch.empty_like(st)


@torch.library.custom_op("alpa_b200::add_layer_norm", mutates_args=())
def add_layer_norm(x: Tensor, r: Tensor, g: Tensor, b: Tensor, eps: float) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """s = x + r; (layer_norm(s), s, mean, rstd) in one pass."""
    if uses_native(x, r, g, b) and x.shape[-1] % 8 == 0 and x.shape[-1] <= 8192:
        y, mean, rstd, s = _native().layernorm_fwd(x.contiguous(), r.contiguous(), g, b, eps, True)
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
    if uses_native(dy, x, g) and H % 8 == 0 and H <= 8192:
        dg = torch.zeros(H, device=x.device, dtype=torch.float32)
        db = torch.zeros(H, device=x.device, dtype=torch.float32)
        dx = _native().layernorm_bwd(dy.contiguous(), x.contiguous(), g, mean.reshape(-1).contiguous(),
                                     rstd.reshape(-1).contiguous(),
                                     dres.contiguous() if dres is not None else None, dg, db)
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


@torch.library.custom_op("alpa_b200::attention", mutates_args=())
def attention(q: Tensor, k: Tensor, v: Tensor, scale: float, causal: bool) -> Tuple[Tensor, Tensor]:
    """(o [B,S,h,D], lse [B,h,S]) = softmax(q k^T * scale [+ causal mask]) v"""
    if uses_native(q, k, v) and q.shape[-1] % 8 == 0 and q.shape[-1] <= 128 and q.stride(-1) == 1:
        o, lse = _native().attention_fwd(q, k, v, scale, causal)
        return o, lse
    return _attn_ref(q, k, v, scale, causal)


@attention.register_fake
def _(q, k, v, scale, causal):
    B, S, H, D = q.shape
    return q.new_empty(B, S, H, D), q.new_empty(B, H, S, dtype=torch.float32)


@torch.library.custom_op("alpa_b200::attention_bwd", mutates_args=())
def attention_bwd(do: Tensor, q: Tensor, k: Tensor, v: Tensor, o: Tensor, lse: Tensor, scale: float,
                  causal: bool) -> Tuple[Tensor, Tensor, Tensor]:
    if uses_native(do, q, k, v, o) and q.shape[-1] % 8 == 0 and q.shape[-1] <= 128 and q.stride(-1) == 1:
        dq, dk, dv = _native().attention_bwd(do, q, k, v, o, lse, scale, causal)
        return dq, dk, dv
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


@attention_bwd.register_fake
def _(do, q, k, v, o, lse, scale, causal):
    return (q.new_empty(q.shape), k.new_empty(k.shape), v.new_empty(v.shape))


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



# ---- packed variant: qkv is one [B, S, heads, 3, D] tensor (a view of the fused QKV projection whose
# output features are ordered (head, {q,k,v}, D) so that a contiguous split of the feature dim is a
# split over heads -- the Megatron layout).  Forward and backward touch the projection output /
# gradient in place: no split/concat copies.
@torch.library.custom_op("alpa_b200::attention_qkvpacked", mutates_args=())
def attention_qkvpacked(qkv: Tensor, scale: float, causal: bool) -> Tuple[Tensor, Tensor]:
    q, k, v = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
    if uses_native(qkv) and qkv.shape[-1] % 8 == 0 and qkv.shape[-1] <= 128 and qkv.stride(-1) == 1:
        o, lse = _native().attention_fwd(q, k, v, scale, causal)
        return o, lse
    return _attn_ref(q, k, v, scale, causal)


@attention_qkvpacked.register_fake
def _(qkv, scale, causal):
    B, S, H, _, D = qkv.shape
    return qkv.new_empty(B, S, H, D), qkv.new_empty(B, H, S, dtype=torch.float32)


@torch.library.custom_op("alpa_b200::attention_qkvpacked_bwd", mutates_args=())
def attention_qkvpacked_bwd(do: Tensor, qkv: Tensor, o: Tensor, lse: Tensor, scale: float, causal: bool) -> Tensor:
    q, k, v = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
    dqkv = torch.empty(qkv.shape, device=qkv.device, dtype=qkv.dtype)
    if uses_native(do, qkv, o) and qkv.shape[-1] % 8 == 0 and qkv.shape[-1] <= 128 and qkv.stride(-1) == 1:
        _native().attention_bwd(do, q, k, v, o, lse, scale, causal, dqkv[:, :, :, 0], dqkv[:, :, :, 1],
                                dqkv[:, :, :, 2])
        return dqkv
    dq, dk, dv = attention_bwd(do, q, k, v, o, lse, scale, causal)
    dqkv[:, :, :, 0], dqkv[:, :, :, 1], dqkv[:, :, :, 2] = dq, dk, dv
    return dqkv


@attention_qkvpacked_bwd.register_fake
def _(do, qkv, o, lse, scale, causal):
    return torch.empty_like(qkv)


def _attn_packed_setup(ctx, inputs, output):
    ctx.set_materialize_grads(False)  # unused outputs yield None, not a zero tensor + add
    qkv, scale, causal = inputs
    o, lse = output
    ctx.save_for_backward(qkv, o, lse)
    ctx.scale, ctx.causal = scale, causal


def _attn_packed_bwd(ctx, do, dlse):
    if do is None:
        return None, None, None
    qkv, o, lse = ctx.saved_tensors
    return attention_qkvpacked_bwd(do, qkv, o, lse, ctx.scale, ctx.causal), None, None


attention_qkvpacked.register_autograd(_attn_packed_bwd, setup_context=_attn_packed_setup)

# =================================================================================================
# embedding (token gather [+ position]) -- the reference lowers this to a one-hot matmul
# (alpa/monkey_patch.py:241-261) to make the vocab dim shardable; we keep a real gather and give the
# planner a vocab-parallel (masked gather + all-reduce) strategy instead.
# =================================================================================================
@torch.library.custom_op("alpa_b200::embedding", mutates_args=())
def embedding(ids: Tensor, wte: Tensor, vocab_start: int = 0) -> Tensor:
    """x[..., H] = wte[ids - vocab_start] (zeros for ids outside this vocab shard)"""
    V = wte.shape[0]
    if uses_native(wte) and wte.shape[1] % 8 == 0:
        return _native().embedding_fwd(ids.contiguous(), None, wte.contiguous(), None, vocab_start)
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
    if uses_native(dy) and H % 2 == 0:
        dt = torch.zeros(num_rows, H, device=dy.device, dtype=torch.float32)
        _native().embedding_bwd_(ids.contiguous(), dy.contiguous(), dt, vocab_start)
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
# decode attention over a KV cache whose valid length lives on the device (serving; not differentiable)
# =================================================================================================
def attention_decode(q: Tensor, k_cache: Tensor, v_cache: Tensor, kv_len: Tensor, scale: float) -> Tensor:
    """q: [B, T, h, D] (the last T positions); k/v_cache: [B, S_max, h, D]; kv_len: int32 scalar tensor = number of
    valid cache rows (including the T new ones).  Causal inside the new block.  Because the length is read on the
    device, one captured CUDA graph serves every decode position."""
    if uses_native(q, k_cache, v_cache):
        return _native().attention_fwd(q if q.stride(-1) == 1 else q.contiguous(), k_cache, v_cache, scale, True,
                                       kv_len)[0]
    n = int(kv_len)
    return _attn_ref(q, k_cache[:, :n], v_cache[:, :n], scale, True)[0]


def decode_attention(q: Tensor, k_new: Tensor, v_new: Tensor, k_cache: Tensor, v_cache: Tensor, kv_len: Tensor,
                     scale: float) -> Tensor:
    """One new token per sequence with the cache append fused in.  q / k_new / v_new: [B, 1, h, D] (views of the fused
    QKV projection are fine); k/v_cache: [B, S_max, h, D], updated in place at row kv_len-1; kv_len: int32 scalar tensor
    = valid rows including the new one.  Returns o [B, 1, h, D].  Replaces two strided copies, two index_copy launches
    and the padded tensor-core attention of `attention_decode` with one cache-streaming kernel."""
    if uses_native(q, k_cache, v_cache) and hasattr(_native(), "decode_attention"):
        if k_new.stride() != v_new.stride() or k_new.stride(-1) != 1:      # e.g. k went through rotary, v did not
            k_new, v_new = k_new.contiguous(), v_new.contiguous()
        return _native().decode_attention(q if q.stride(-1) == 1 else q.contiguous(), k_new, v_new, k_cache, v_cache,
                                          kv_len, scale)
    n = int(kv_len)
    k_cache[:, n - 1:n] = k_new
    v_cache[:, n - 1:n] = v_new
    return _attn_ref(q, k_cache[:, :n], v_cache[:, :n], scale, True)[0]


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
    if uses_native(q, k_cache, v_cache) and q.shape[-1] % 8 == 0 and q.shape[-1] <= 128:
        if T == 1 and hasattr(_native(), "decode_attention"):
            kv_len = (cache_len.to(torch.int32) + 1).reshape(())
            return decode_attention(q, k_new, v_new, k_cache, v_cache, kv_len, scale)
        # prompt chunk: same kernel path as the serving decoder's prefill (flash attention over the valid cache rows,
        # causal with Sq != Sk); the length is read on the host here -- only the T = 1 step has to be sync-free
        n0 = int(cache_len)
        k_cache[:, n0:n0 + T] = k_new
        v_cache[:, n0:n0 + T] = v_new
        return attention(q if q.stride(-1) == 1 else q.contiguous(), k_cache[:, :n0 + T], v_cache[:, :n0 + T], scale,
                         True)[0]
    n0 = int(cache_len)
    k_cache[:, n0:n0 + T] = k_new
    v_cache[:, n0:n0 + T] = v_new
    return _attn_ref(q, k_cache[:, :n0 + T], v_cache[:, :n0 + T], scale, True)[0]


# =================================================================================================
# attention of a ragged 1-D token batch over a slot-addressed KV cache (iteration-level batching; not differentiable)
# =================================================================================================
def ragged_attention(q: Tensor, k_cache: Tensor, v_cache: Tensor, seq_start: Tensor, ctx_len: Tensor, scale: float,
                     max_ctx: int, alibi: Optional[Tensor] = None) -> Tensor:
    """q: [T, h, D]; k/v_cache: [slots, h, D]; token t attends to cache rows seq_start[t] .. seq_start[t]+ctx_len[t]-1
    (ctx_len 0 = padding token -> zeros).  `max_ctx` bounds ctx_len (sizes the score buffer).  `alibi`: optional fp32
    [h] slopes, bias = slope * key position.  (reference: the external fused_mmha of opt_model_1d.py:151-178)"""
    if uses_native(q, k_cache, v_cache):
        return _native().ragged_attention(q if q.stride(-1) == 1 else q.contiguous(), k_cache, v_cache, seq_start,
                                          ctx_len, scale, max_ctx, alibi)
    T, h, D = q.shape
    longest = int(ctx_len.max()) if T else 0
    if longest > max_ctx:
        # the kernel's score buffer holds max_ctx keys; clamping would silently drop the newest keys
        raise ValueError(f"ragged_attention: ctx_len {longest} exceeds max_ctx {max_ctx}")
    n = longest
    if n == 0:
        return torch.zeros_like(q)
    j = torch.arange(n, device=q.device)
    idx = (seq_start.long()[:, None] + j[None, :]).clamp_(max=k_cache.shape[0] - 1)          # [T, n]
    k = k_cache[idx].float()                                                                     # [T, n, h, D]
    v = v_cache[idx].float()
    s = torch.einsum("thd,tnhd->thn", q.float() * scale, k)
    if alibi is not None:
        s = s + alibi.view(1, h, 1) * j.view(1, 1, n)
    valid = j[None, :] < ctx_len.long()[:, None]                                                 # [T, n]
    s = s.masked_fill(~valid[:, None, :], float("-inf"))
    p = torch.softmax(s, dim=-1)
    p = torch.nan_to_num(p, nan=0.0)                                                             # padding rows
    return torch.einsum("thn,tnhd->thd", p, v).to(q.dtype)


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
    if x.is_cuda and 1 <= x.dim() <= 6 and x.dtype in (torch.bfloat16, torch.float32) and \
            (uses_native(x) or (x.dtype == torch.float32 and uses_native(x.new_empty(0, dtype=torch.bfloat16)))):
        return _native().dropout(x, float(p), seed.to(x.device), int(stream), list(global_shape), list(offsets))
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
def linear_decode(x: Tensor, w: Tensor, w_scale: Optional[Tensor], b: Optional[Tensor] = None, act: str = "none",
                  residual: Optional[Tensor] = None, ln: Optional[Tuple[Tensor, Tensor, float]] = None) -> Tensor:
    """y = act(LN(x) @ W^T * w_scale + b) (+ residual) for a handful of tokens (decode): weight-streaming GEMV on
    sm_90a (the streamed fp8 / bf16 weight bytes go to the tensor cores unconverted; with fp8 weights the activations
    are quantised per token to e4m3 inside the kernel, like the prefill fp8 GEMM; no tile padding); not
    differentiable.  x: [..., K] with at most 8 rows in total.  `ln` = (gamma, beta, eps) layer-normalises x inside the
    kernel's prologue (one launch less per projection); None = x is used as is."""
    rows = x.numel() // x.shape[-1]
    K = x.shape[-1]
    if x.is_cuda and global_config.use_native_kernels and rows <= 8 and x.dtype == torch.bfloat16:
        from alpa_b200 import ops
        fp8w = w.dtype == torch.float8_e4m3fn
        if ops.native_available() and hasattr(_native(), "gemv_decode") and K % (64 if fp8w else 32) == 0 and \
                rows * K * (1 if fp8w else 2) <= 200 * 1024:
            x2 = _as2d(x)
            if x2.stride(0) % 8 or x2.data_ptr() % 16:     # the prologue reads rows 16 bytes at a time
                x2 = x2.contiguous()
            r2 = None if residual is None else _as2d(residual)
            if ln is not None and ln[0].dtype != torch.bfloat16:
                x2 = layer_norm(x2, ln[0], ln[1], ln[2])[0]          # the fused prologue reads bf16 gamma / beta
                ln = None
            if ln is None:
                y = _native().gemv_decode(x2, w, w_scale, b, r2, _ACT_IDS[act])
            else:
                y = _native().gemv_decode(x2, w, w_scale, b, r2, _ACT_IDS[act], ln[0], ln[1], float(ln[2]))
            return y.view(*x.shape[:-1], w.shape[0])
    if ln is not None:
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
    if x.is_cuda and global_config.use_native_kernels:
        from alpa_b200 import ops
        if ops.native_available() and hasattr(_native(), "gemm_fp8") and x.shape[-1] % 16 == 0 and w_fp8.shape[0] % 8 == 0:
            x2 = _as2d(x)
            if x2.stride(0) % 8 or x2.data_ptr() % 16:     # the quantiser reads rows 16 bytes at a time
                x2 = x2.contiguous()
            y = _native().gemm_fp8(x2, w_fp8, w_scale, b, _ACT_IDS[act])
            return y.view(*x.shape[:-1], w_fp8.shape[0])
    w = (w_fp8.to(torch.float32) * w_scale[:, None]).to(x.dtype)
    y = F.linear(x, w, b)
    return _act_fn(y, act)


# =================================================================================================
# cross-mesh resharding pack / unpack: the tiles one device exchanges with a peer as ONE contiguous message
# =================================================================================================
def packed_nbytes(views: List[Tensor]) -> int:
    """Bytes of the staging buffer of `views` (every tile starts on a 16-byte boundary)."""
    return sum((v.numel() * v.element_size() + 15) // 16 * 16 for v in views)


def _pack_native_ok(views: List[Tensor], flat: Tensor) -> bool:
    return (flat.is_cuda and global_config.use_native_kernels and hasattr(_native(), "pack_tiles") and
            all(v.is_cuda and 1 <= v.dim() <= 4 and v.stride(-1) == 1 and v.numel() > 0 for v in views))


def pack_tiles(views: List[Tensor], flat: Optional[Tensor] = None) -> Tensor:
    """Gather strided slices into one uint8 staging buffer (one launch on sm_90a: pack_sm90.cu)."""
    if flat is None:
        flat = torch.empty(packed_nbytes(views), dtype=torch.uint8, device=views[0].device)
    if views and _pack_native_ok(views, flat):
        _native().pack_tiles(list(views), flat, False)
        return flat
    off = 0
    for v in views:
        n = v.numel() * v.element_size()
        flat[off:off + n].copy_(v.contiguous().view(-1).view(torch.uint8))
        off += (n + 15) // 16 * 16
    return flat


def unpack_tiles(flat: Tensor, views: List[Tensor]) -> None:
    """Scatter a received staging buffer into the destination slices (in place)."""
    if views and _pack_native_ok(views, flat):
        _native().pack_tiles(list(views), flat, True)
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
    if uses_native(x) and hasattr(_native(), "quantize_mxfp8"):
        ok = x.stride(-1) == 1 and x.stride(0) % 8 == 0 and x.data_ptr() % 16 == 0
        q, sf = _native().quantize_mxfp8(x if ok else x.contiguous())
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
    if uses_native(x) and hasattr(_native(), "gemm_mxfp8") and K % MX_BLOCK == 0 and N % 8 == 0:
        if x2.stride(0) % 8 or x2.data_ptr() % 16:         # the quantiser reads rows 16 bytes at a time
            x2 = x2.contiguous()
        y = _native().gemm_mxfp8(x2, w_q, w_sf, b, _ACT_IDS[act])
        return y.view(*x.shape[:-1], N)
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
    if uses_native(a, b) and _gemm_ok(a, b):
        return _native().gemm(a, b, trans_a, trans_b)
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
    C = capacity
    if gates.is_cuda and global_config.use_native_kernels:
        from alpa_b200 import ops
        if ops.native_available():
            return tuple(_native().moe_top2_route(gates.float().contiguous(), C))
        if not ops.allow_fallback():
            raise RuntimeError("alpa_b200: sm_90a extension missing for moe_top2_route")
    idx1 = gates.argmax(-1)
    mask1 = F.one_hot(idx1, E)
    idx2 = (gates * (1 - mask1)).argmax(-1)
    mask2 = F.one_hot(idx2, E)
    pos1_all = mask1.cumsum(-2) - mask1
    keep1 = (pos1_all < C) & mask1.bool()
    pos1 = (pos1_all * keep1).sum(-1)
    ok1 = keep1.any(-1)
    count1 = keep1.sum(-2)
    pos2_all = (mask2.cumsum(-2) - mask2) + count1.unsqueeze(-2)
    keep2 = (pos2_all < C) & mask2.bool()
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
    if uses_native(x, weight) and M % 8 == 0:
        d = torch.zeros(num_experts, G * capacity, M, device=x.device, dtype=x.dtype)
        _native().moe_dispatch_(x.contiguous(), expert.contiguous(), slot.contiguous(),
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
    C = GC // G
    if uses_native(eo, weight) and M % 8 == 0:
        return _native().moe_combine(eo.contiguous(), expert.contiguous(), slot.contiguous(),
                                     None if weight is None else weight.contiguous())
    g = torch.arange(G, device=eo.device).view(G, 1, 1)
    ok = slot >= 0
    row = torch.where(ok, (expert * G + g) * C + slot, torch.zeros_like(slot))
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
    C = GC // G
    if uses_native(eo, dout) and M % 8 == 0:
        return _native().moe_combine_wgrad(dout.contiguous(), eo.contiguous(), expert.contiguous(),
                                           slot.contiguous())
    g = torch.arange(G, device=eo.device).view(G, 1, 1)
    ok = slot >= 0
    row = torch.where(ok, (expert * G + g) * C + slot, torch.zeros_like(slot))
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
    if uses_native(logits) and V % 8 == 0 and l2.stride(0) % 8 == 0 and l2.stride(1) == 1:
        stats = _native().ce_stats(l2, lab.contiguous(), vocab_start)
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
    if uses_native(logits) and V % 8 == 0:
        g = logits.reshape(T, V).clone()
        _native().ce_grad_(g, lab.contiguous(), stats[:, :2].contiguous(),
                           dloss.reshape(T).float().contiguous(), vocab_start)
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
    if masters and masters[0].is_cuda and global_config.use_native_kernels:
        from alpa_b200 import ops
        if ops.native_available() and all(g.dtype in (torch.float32, torch.bfloat16) for g in grads):
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
                tab = _native().adam_build_tables(gsrc, masters, ms, vs, pb, list(weight_decays))
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
            _native().adamw_step(tab[0], tab[1], lr, beta1, beta2, eps, 1, grad_scale, None,
                                 step.float().reshape(1))
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
    if uses_native(dy, x) and out.dtype == torch.bfloat16:
        d2, x2 = _as2d(dy), _as2d(x)
        if _gemm_ok(d2, x2) and out.stride(-1) == 1 and out.data_ptr() % 16 == 0 and out.stride(0) % 8 == 0:
            _native().gemm(d2, x2, True, True, out=out)
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
        self.attention_decode = attention_decode
        self.decode_attention = decode_attention
        self.ragged_attention = ragged_attention
        self.linear_mxfp8 = linear_mxfp8


fast = _FastNamespace(_fast_ns)
__all__ += ["DIRECT_IMPL", "DIRECT_OUT_IMPL", "INPLACE_IMPL", "fast"]
