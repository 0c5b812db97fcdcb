"""Train state, functional optimizers and mixed-precision helpers.

Reference: alpa/model/model_util.py (TrainState:273-378 with fp32 master copy, DynamicScale:381-491)
and the optax transformations the reference benchmarks use (adamw / adafactor / sgd).  Everything here
is a torch pytree of tensors plus static configuration, so a whole train step -- forward, backward
and the update -- traces into one graph.
"""
from __future__ import annotations

import math

from dataclasses import dataclass
from typing import Any, Callable, Dict, Optional

import torch
from torch.utils import _pytree as pytree

from alpa_b200.ops.primitives import fused_adamw_


# ------------------------------------------------------------------------------------------------
# functional optimizers (optax-like GradientTransformation: init / update)
# ------------------------------------------------------------------------------------------------
class Optimizer:
    def init(self, params):
        raise NotImplementedError

    def update(self, grads, opt_state, params, step):
        """-> (new_params, new_opt_state); `step` is the 1-based step count (float tensor)."""
        raise NotImplementedError


def _tmap(f, *trees):
    return pytree.tree_map(f, *trees)


# ------------------------------------------------------------------------------------------------
# learning-rate schedules: callables step (1-based float tensor) -> lr, written in traceable tensor math so that the
# schedule is part of the compiled step (reference examples use optax.linear_schedule / join_schedules /
# warmup_cosine_decay_schedule, e.g. examples/gpt2/run_clm_flax.py, examples/opt_finetune/run_clm_flax.py)
# ------------------------------------------------------------------------------------------------
def constant_schedule(value: float):
    return lambda step: step * 0.0 + value


def linear_schedule(init_value: float, end_value: float, transition_steps: int, transition_begin: int = 0):
    def fn(step):
        frac = torch.clamp((step - transition_begin) / max(1, transition_steps), 0.0, 1.0)
        return init_value + (end_value - init_value) * frac
    return fn


def cosine_decay_schedule(init_value: float, decay_steps: int, alpha: float = 0.0):
    def fn(step):
        frac = torch.clamp(step / max(1, decay_steps), 0.0, 1.0)
        return init_value * ((1 - alpha) * 0.5 * (1 + torch.cos(math.pi * frac)) + alpha)
    return fn


def join_schedules(schedules, boundaries):
    """schedules[i] is active between boundaries[i-1] and boundaries[i]; each sees the step count relative to the
    start of its own interval."""
    assert len(schedules) == len(boundaries) + 1

    def fn(step):
        out = schedules[0](step)
        for b, sch in zip(boundaries, schedules[1:]):
            out = torch.where(step < b, out, sch(step - b))
        return out
    return fn


def warmup_cosine_decay_schedule(init_value: float, peak_value: float, warmup_steps: int, decay_steps: int,
                                 end_value: float = 0.0):
    alpha = end_value / peak_value if peak_value else 0.0
    return join_schedules([linear_schedule(init_value, peak_value, warmup_steps),
                           cosine_decay_schedule(peak_value, max(1, decay_steps - warmup_steps), alpha)], [warmup_steps])


def _lr_at(lr, step):
    return lr(step) if callable(lr) else lr


class SGD(Optimizer):
    def __init__(self, learning_rate: float, momentum: float = 0.0, weight_decay: float = 0.0):
        self.lr, self.momentum, self.weight_decay = learning_rate, momentum, weight_decay

    def init(self, params):
        if self.momentum == 0.0:
            return {}
        return {"trace": _tmap(lambda p: torch.zeros_like(p, dtype=torch.float32), params)}

    def update(self, grads, opt_state, params, step):
        wd = self.weight_decay
        lr = _lr_at(self.lr, step)
        if self.momentum == 0.0:
            new = _tmap(lambda p, g: (p.float() - lr * (g.float() + wd * p.float())).to(p.dtype), params, grads)
            return new, opt_state
        trace = _tmap(lambda t, g, p: self.momentum * t + g.float() + wd * p.float(), opt_state["trace"], grads, params)
        new = _tmap(lambda p, t: (p.float() - lr * t).to(p.dtype), params, trace)
        return new, {"trace": trace}


class Adam(Optimizer):
    """Adam / AdamW on fp32 state.  fused=True runs the single-launch sm_90a multi-tensor kernel in
    place (requires the train state to be donated); fused=False is plain traceable torch math."""

    def __init__(self, learning_rate: float, b1: float = 0.9, b2: float = 0.999, eps: float = 1e-8,
                 weight_decay: float = 0.0, mask: Optional[Callable] = None, fused: bool = False):
        self.lr, self.b1, self.b2, self.eps = learning_rate, b1, b2, eps
        self.weight_decay, self.mask, self.fused = weight_decay, mask, fused

    def init(self, params):
        return {"mu": _tmap(lambda p: torch.zeros_like(p, dtype=torch.float32), params),
                "nu": _tmap(lambda p: torch.zeros_like(p, dtype=torch.float32), params)}

    def _decays(self, params):
        leaves = pytree.tree_leaves(params)
        if self.weight_decay == 0.0:
            return [0.0] * len(leaves)
        if self.mask is None:
            return [self.weight_decay] * len(leaves)
        m = pytree.tree_leaves(self.mask(params))
        return [self.weight_decay if bool(x) else 0.0 for x in m]

    def update(self, grads, opt_state, params, step, master=None):
        p_leaves, tree = pytree.tree_flatten(params)
        g_leaves = pytree.tree_leaves(grads)
        mu = pytree.tree_leaves(opt_state["mu"])
        nu = pytree.tree_leaves(opt_state["nu"])
        w_leaves = pytree.tree_leaves(master) if master is not None else p_leaves
        wds = self._decays(params)
        if self.fused:
            if callable(self.lr):
                raise ValueError("the fused AdamW kernel takes a constant learning rate; use fused=False with a schedule")
            fused_adamw_(p_leaves, w_leaves, mu, nu, g_leaves, step, self.lr, self.b1, self.b2, self.eps, wds, 1.0)
            return params, opt_state, master
        lr = _lr_at(self.lr, step)
        bc1 = 1.0 - self.b1 ** step
        bc2 = 1.0 - self.b2 ** step
        new_p, new_w, new_mu, new_nu = [], [], [], []
        for p, w, m, v, g, wd in zip(p_leaves, w_leaves, mu, nu, g_leaves, wds):
            gf = g.float()
            m2 = self.b1 * m + (1 - self.b1) * gf
            v2 = self.b2 * v + (1 - self.b2) * gf * gf
            upd = (m2 / bc1) / (torch.sqrt(v2 / bc2) + self.eps)
            if wd != 0.0:
                upd = upd + wd * w.float()
            w2 = w.float() - lr * upd
            new_w.append(w2.to(w.dtype))
            new_p.append(w2.to(p.dtype))
            new_mu.append(m2)
            new_nu.append(v2)
        new_params = pytree.tree_unflatten(new_p, tree)
        new_state = {"mu": pytree.tree_unflatten(new_mu, tree), "nu": pytree.tree_unflatten(new_nu, tree)}
        new_master = pytree.tree_unflatten(new_w, tree) if master is not None else None
        return new_params, new_state, new_master


def sgd(learning_rate, momentum=0.0, weight_decay=0.0):
    return SGD(learning_rate, momentum, weight_decay)


def adam(learning_rate, b1=0.9, b2=0.999, eps=1e-8, fused=False):
    return Adam(learning_rate, b1, b2, eps, 0.0, None, fused)


def adamw(learning_rate, b1=0.9, b2=0.999, eps=1e-8, weight_decay=1e-4, mask=None, fused=False):
    return Adam(learning_rate, b1, b2, eps, weight_decay, mask, fused)


class Adafactor(Optimizer):
    """Factored second-moment optimizer used by the reference's MoE benchmark
    (benchmark/alpa/benchmark_one_case_moe.py:29, optax.adafactor): row/column statistics for
    matrices, full statistics for vectors; update clipping by RMS; no momentum."""

    def __init__(self, learning_rate: float, decay_rate: float = 0.8, eps: float = 1e-30, clip: float = 1.0,
                 min_dim_size_to_factor: int = 128):
        self.lr, self.decay_rate, self.eps, self.clip = learning_rate, decay_rate, eps, clip
        self.min_dim = min_dim_size_to_factor

    def _factored(self, p):
        return p.dim() >= 2 and p.shape[-1] >= self.min_dim and p.shape[-2] >= self.min_dim

    def init(self, params):
        def one(p):
            if self._factored(p):
                return {"vr": torch.zeros(p.shape[:-1], dtype=torch.float32, device=p.device),
                        "vc": torch.zeros(p.shape[:-2] + p.shape[-1:], dtype=torch.float32, device=p.device)}
            return {"v": torch.zeros_like(p, dtype=torch.float32)}
        leaves, tree = pytree.tree_flatten(params)
        return {"stats": [one(p) for p in leaves]}

    def update(self, grads, opt_state, params, step, master=None):
        p_leaves, tree = pytree.tree_flatten(params)
        g_leaves = pytree.tree_leaves(grads)
        beta2 = 1.0 - torch.pow(step, -self.decay_rate)
        new_p, new_stats = [], []
        for p, g, st in zip(p_leaves, g_leaves, opt_state["stats"]):
            gf = g.float()
            g2 = gf * gf + self.eps
            if "vr" in st:
                vr = beta2 * st["vr"] + (1 - beta2) * g2.mean(-1)
                vc = beta2 * st["vc"] + (1 - beta2) * g2.mean(-2)
                r = vr / vr.mean(-1, keepdim=True)
                u = gf * torch.rsqrt(r.unsqueeze(-1)) * torch.rsqrt(vc.unsqueeze(-2))
                new_stats.append({"vr": vr, "vc": vc})
            else:
                v = beta2 * st["v"] + (1 - beta2) * g2
                u = gf * torch.rsqrt(v)
                new_stats.append({"v": v})
            rms = torch.sqrt((u * u).mean())
            u = u / torch.clamp(rms / self.clip, min=1.0)
            new_p.append((p.float() - _lr_at(self.lr, step) * u).to(p.dtype))
        return pytree.tree_unflatten(new_p, tree), {"stats": new_stats}, master


def adafactor(learning_rate, **kw):
    return Adafactor(learning_rate, **kw)


# ------------------------------------------------------------------------------------------------
# dynamic loss scale (reference: DynamicScale, model_util.py:381-491)
# ------------------------------------------------------------------------------------------------
@dataclass
class DynamicScale:
    growth_factor: float = 2.0
    backoff_factor: float = 0.5
    growth_interval: int = 2000
    fin_steps: Any = None   # tensor scalar
    scale: Any = None       # tensor scalar

    @staticmethod
    def create(init_scale: float = 65536.0, device="cpu"):
        return DynamicScale(fin_steps=torch.zeros((), device=device), scale=torch.tensor(float(init_scale), device=device))

    def update(self, grads):
        """-> (new DynamicScale, is_finite scalar bool tensor, unscaled grads)"""
        leaves, tree = pytree.tree_flatten(grads)
        finite = torch.stack([torch.isfinite(g.float()).all() for g in leaves]).all()
        grow = self.fin_steps + 1 >= self.growth_interval
        new_scale = torch.where(finite, torch.where(grow, self.scale * self.growth_factor, self.scale),
                                self.scale * self.backoff_factor)
        new_fin = torch.where(finite & ~grow, self.fin_steps + 1, torch.zeros_like(self.fin_steps))
        unscaled = pytree.tree_unflatten([g / self.scale for g in leaves], tree)
        return DynamicScale(self.growth_factor, self.backoff_factor, self.growth_interval, new_fin, new_scale), finite, unscaled


pytree.register_pytree_node(
    DynamicScale,
    lambda d: ([d.fin_steps, d.scale], (d.growth_factor, d.backoff_factor, d.growth_interval)),
    lambda ch, ctx: DynamicScale(ctx[0], ctx[1], ctx[2], ch[0], ch[1]))


# ------------------------------------------------------------------------------------------------
# TrainState
# ------------------------------------------------------------------------------------------------
class TrainState:
    """Parameters + optimizer state (+ optional fp32 master copy) as one pytree.

    Reference: alpa/model/model_util.py:273-378.  `params` are in the compute dtype (bf16 on the GPU);
    with `use_master_copy` the optimizer runs on `master_copy` (fp32) and refreshes `params`."""

    def __init__(self, step, params, opt_state, master_copy=None, dynamic_scale=None, apply_fn=None, tx=None):
        self.step = step
        self.params = params
        self.opt_state = opt_state
        self.master_copy = master_copy
        self.dynamic_scale = dynamic_scale
        self.apply_fn = apply_fn
        self.tx = tx

    @classmethod
    def create(cls, *, apply_fn, params, tx: Optimizer, use_master_copy: bool = False, dynamic_scale=None):
        first = pytree.tree_leaves(params)[0]
        master = None
        if use_master_copy:
            master = pytree.tree_map(lambda p: p.detach().float().clone(), params)
        opt_state = tx.init(master if master is not None else params)
        step = torch.zeros((), dtype=torch.float32, device=first.device)
        return cls(step, params, opt_state, master, dynamic_scale, apply_fn, tx)

    def apply_gradients(self, *, grads, **kwargs):
        step = self.step + 1
        if isinstance(self.tx, (Adam, Adafactor)):
            new_params, new_opt, new_master = self.tx.update(grads, self.opt_state, self.params, step,
                                                             master=self.master_copy)
        else:
            target = self.master_copy if self.master_copy is not None else self.params
            new_target, new_opt = self.tx.update(grads, self.opt_state, target, step)
            if self.master_copy is not None:
                new_master = new_target
                new_params = pytree.tree_map(lambda w, p: w.to(p.dtype), new_target, self.params)
            else:
                new_master, new_params = None, new_target
        return TrainState(step, new_params, new_opt, new_master, kwargs.get("dynamic_scale", self.dynamic_scale),
                          self.apply_fn, self.tx)

    def replace(self, **kw):
        d = dict(step=self.step, params=self.params, opt_state=self.opt_state, master_copy=self.master_copy,
                 dynamic_scale=self.dynamic_scale, apply_fn=self.apply_fn, tx=self.tx)
        d.update(kw)
        return TrainState(**d)


def _ts_flatten(s: TrainState):
    return [s.step, s.params, s.opt_state, s.master_copy, s.dynamic_scale], (s.apply_fn, s.tx)


def _ts_unflatten(children, ctx):
    return TrainState(children[0], children[1], children[2], children[3], children[4], ctx[0], ctx[1])


pytree.register_pytree_node(TrainState, _ts_flatten, _ts_unflatten)


def functional_call(module: torch.nn.Module, params: Dict[str, torch.Tensor], args=(), kwargs=None,
                    method: Optional[str] = None):
    """Run `module` with `params` substituted (the analogue of flax's `apply_fn(params, ...)`).  `method` names a
    method other than `forward` (flax: `apply(..., method=...)`)."""
    if method is None:
        return torch.func.functional_call(module, params, args, kwargs or {})
    from torch.nn.utils.stateless import _reparametrize_module
    with _reparametrize_module(module, params):
        return getattr(module, method)(*args, **(kwargs or {}))


def params_of(module: torch.nn.Module) -> Dict[str, torch.Tensor]:
    return {k: v.detach() for k, v in module.named_parameters()}


def is_tensor(x) -> bool:
    """(reference: model_util.is_tensor)"""
    return isinstance(x, torch.Tensor) or hasattr(x, "sharding_spec")


def softmax_cross_entropy(logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """Cross entropy against soft / one-hot label distributions: -sum(labels * log_softmax(logits)) over the last
    dim (reference: model_util.softmax_cross_entropy:269-270)."""
    return -(labels * torch.log_softmax(logits.float(), dim=-1)).sum(dim=-1)
