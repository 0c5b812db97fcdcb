"""Layer construction: cut the forward computation into pipeline layers.

Reference: alpa/pipeline_parallel/layer_construction.py (ManualLayerOption:46, AutoLayerOption:70,
FollowLayerOption:121, cluster_jaxpr_by_cost:342, automatic_layer_construction:650, manual_remat /
automatic_remat:542-692) and layer_stats.py (eqn_flops:12, heavy_count:49).

The reference transforms the forward jaxpr before differentiation so that the marker's transpose rule
creates the backward boundaries.  Here the same effect is obtained with torch machinery: a
``TorchFunctionMode`` watches the *heavy* operators (linear / matmul / conv / attention) while the
forward function runs under tracing and routes the result of the op chosen as a cut point through
``mark_pipeline_boundary``; autograd then emits the mirrored backward marker.  Cut points come from a
first profiling pass of the same function and the native clustering DP (``cluster_ops_by_cost``).
"""
from __future__ import annotations

import functools

import logging
from abc import ABC
from typing import Callable, List, Optional, Sequence

import torch
import torch.nn.functional as F
from torch.overrides import TorchFunctionMode

from alpa_b200.global_env import global_config
from alpa_b200.parallel.pipeline.primitive_def import mark_pipeline_boundary

logger = logging.getLogger(__name__)


class LayerOption(ABC):
    """Options of layer construction (reference: layer_construction.py:31-43)."""

    def __init__(self):
        self.layer_num: Optional[int] = None

    def transform(self, func: Callable) -> Callable:
        return func


class ManualLayerOption(LayerOption):
    """The user (or the model, e.g. GPTConfig.add_manual_pipeline_markers) placed
    ``mark_pipeline_boundary`` calls (reference: layer_construction.py:46-67)."""

    def __init__(self, remat_layer: bool = False, static_argnums: Sequence[int] = ()):
        super().__init__()
        self.remat_layer = remat_layer
        self.static_argnums = static_argnums

    def transform(self, func):
        return func


class AutoLayerOption(LayerOption):
    """Cluster the forward operators into `layer_num` layers of balanced FLOPs with small cuts
    (reference: layer_construction.py:70-118)."""

    def __init__(self, layer_num: int, remat_mode: str = "none", fine_grained_remat_layer_num: Optional[int] = None,
                 static_argnums: Sequence[int] = (), eps: float = 0.6):
        super().__init__()
        self.layer_num = layer_num
        self.remat_mode = remat_mode
        self.fine_grained_remat_layer_num = fine_grained_remat_layer_num
        self.static_argnums = static_argnums
        self.eps = eps

    def transform(self, func):
        if self.remat_mode == "fine_grained_remat" and self.fine_grained_remat_layer_num:
            # finer recomputation segments inside the pipeline layers (markers that do not cut stages)
            from alpa_b200.parallel.pipeline.primitive_def import mark_remat_boundary
            func = automatic_layer_construction(func, self.fine_grained_remat_layer_num, self.eps,
                                                mark=mark_remat_boundary)
        if self.layer_num is None or (self.layer_num != "auto" and self.layer_num <= 1):
            return func
        return automatic_layer_construction(func, self.layer_num, self.eps)


class FollowLayerOption(LayerOption):
    """Follow the layer boundaries implied by the input placement of another executable
    (reference: layer_construction.py:121-157)."""

    def __init__(self, input_placement_specs, num_meshes: int, static_argnums: Sequence[int] = ()):
        super().__init__()
        self.input_placement_specs = input_placement_specs
        self.num_meshes = num_meshes
        self.static_argnums = static_argnums
        self.layer_num = num_meshes


# ------------------------------------------------------------------------------------------------
# heavy-op accounting (reference: layer_stats.py eqn_flops / heavy_count / is_nontrivial)
# ------------------------------------------------------------------------------------------------
def _numel(shape) -> float:
    n = 1.0
    for s in shape:
        n *= s
    return n


def heavy_op_flops(func, args, kwargs, out) -> float:
    """FLOPs of a heavy operator call, 0 for everything else."""
    name = getattr(func, "__name__", str(func))
    full = str(func)
    try:
        if func in (F.linear,) or "alpa_b200.linear" in full and "grad" not in full:
            x, w = args[0], args[1]
            return 2.0 * _numel(x.shape) * w.shape[0]
        if func in (torch.matmul, torch.mm, torch.bmm, torch.Tensor.matmul, torch.Tensor.mm, torch.Tensor.bmm,
                    torch.Tensor.__matmul__):
            a, b = args[0], args[1]
            if a.dim() >= 1 and b.dim() >= 2:
                return 2.0 * _numel(a.shape) * b.shape[-1]
            return 0.0
        if func in (F.conv2d, F.conv1d, F.conv3d):
            w = args[1]
            o = out[0] if isinstance(out, (tuple, list)) else out
            return 2.0 * _numel(o.shape) * _numel(w.shape[1:])
        if "alpa_b200.attention" in full and "bwd" not in full:
            q = args[0]
            if "gqa" in full:                      # [B, S, Hkv, G + 2, D]: G query heads per K/V head
                B, S, Hkv, P, D = q.shape
                H = Hkv * (P - 2)
            elif q.dim() == 5:
                B, S, H, _, D = q.shape
            else:
                B, S, H, D = q.shape
            return 4.0 * B * H * S * S * D
        if func is F.scaled_dot_product_attention:
            q, k = args[0], args[1]
            return 4.0 * _numel(q.shape) * k.shape[-2]
    except Exception:  # noqa: BLE001
        return 0.0
    return 0.0


class _HeavyOpProfiler(TorchFunctionMode):
    """Pass 1: record (flops, output bytes) of each heavy op in execution order."""

    def __init__(self):
        super().__init__()
        self.records: List[tuple] = []
        self.active = True

    def __torch_function__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        out = func(*args, **kwargs)
        if self.active and torch.is_grad_enabled():
            fl = heavy_op_flops(func, args, kwargs, out)
            if fl > 0:
                o = out[0] if isinstance(out, (tuple, list)) else out
                self.records.append((fl, _numel(o.shape) * o.element_size()))
        return out


class _BoundaryInserter(TorchFunctionMode):
    """Pass 2: after the heavy ops listed in `cut_after`, pass the result through a pipeline marker."""

    def __init__(self, cut_after: Sequence[int], mark=None):
        super().__init__()
        self.cut_after = set(cut_after)
        self.count = 0
        self.active = True
        self.mark = mark or mark_pipeline_boundary

    def __torch_function__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        out = func(*args, **kwargs)
        if self.active and torch.is_grad_enabled() and heavy_op_flops(func, args, kwargs, out) > 0:
            idx = self.count
            self.count += 1
            if idx in self.cut_after:
                self.active = False
                try:
                    if isinstance(out, (tuple, list)):
                        first = self.mark(out[0])
                        out = type(out)([first] + list(out[1:]))
                    else:
                        out = self.mark(out)
                finally:
                    self.active = True
        return out


def cluster_heavy_ops(records: Sequence[tuple], layer_num: int, eps: float) -> List[int]:
    """Indices (into the heavy-op sequence) after which a layer boundary is placed."""
    from alpa_b200.parallel.shard.auto_sharding import planner_module
    P = planner_module()
    flops = [r[0] for r in records]
    cut_cost = [r[1] for r in records]
    layer_of = P.cluster_ops_by_cost(flops, cut_cost, int(layer_num), float(eps))
    cuts = [i for i in range(len(layer_of) - 1) if layer_of[i + 1] != layer_of[i]]
    return cuts


def search_layer_num(records: Sequence[tuple], eps: float, layer_eps: float = 0.0) -> int:
    """`layer_num="auto"`: the largest layer count whose clustering does not cut more bytes than the 2-layer
    clustering does (up to a factor 1 + layer_eps), found by bisection between 2 and #heavy-ops / 3 + 1
    (reference: search_layer_num, layer_construction.py:460-487)."""
    n = len(records)
    if n < 2:
        return 1

    def total_cut(k):
        return sum(records[i][1] for i in cluster_heavy_ops(records, k, eps))
    lo, hi = 2, n // 3 + 1
    if hi <= lo:
        return min(lo, n)
    base = total_cut(lo)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if total_cut(mid) > base * (1 + layer_eps) * (mid - 1):      # allow the cut volume to grow with the cut count
            hi = mid
        else:
            lo = mid
    return lo


def automatic_layer_construction(func: Callable, layer_num, eps: float = 0.6, layer_eps: float = 0.0,
                                 mark=None) -> Callable:
    """Wrap `func` (the loss function handed to alpa_b200.grad) so that running it inserts
    `layer_num - 1` pipeline boundaries at FLOP-balanced positions (`layer_num="auto"`: see search_layer_num).
    `mark`: the marker to insert (default: pipeline boundaries; `mark_remat_boundary` for remat-only segments)."""
    state = {"cuts": None}

    def wrapped(*args, **kwargs):
        if state["cuts"] is None:
            prof = _HeavyOpProfiler()
            with torch.no_grad():
                # profile on detached inputs: same shapes, no autograd graph, results discarded
                with torch.enable_grad():
                    with prof:
                        func(*args, **kwargs)
            nonlocal layer_num
            if layer_num == "auto":
                layer_num = search_layer_num(prof.records, eps, layer_eps)
            if len(prof.records) < layer_num:
                logger.warning("auto layer construction: only %d heavy ops for %d layers", len(prof.records), layer_num)
            state["cuts"] = cluster_heavy_ops(prof.records, min(layer_num, max(1, len(prof.records))), eps)
            if global_config.print_auto_layer_stats:
                print(f" - auto layers: {len(prof.records)} heavy ops, cuts after {state['cuts']}")
        with _BoundaryInserter(state["cuts"], mark):
            return func(*args, **kwargs)

    return wrapped


def manual_remat(fun: Optional[Callable] = None, *, static_argnums: Sequence[int] = ()):
    """Recompute each layer (delimited by `mark_pipeline_boundary`) in the backward pass instead of keeping its
    activations (reference: manual_remat, layer_construction.py:542).  Wrap the loss function:
    `alpa.value_and_grad(alpa.manual_remat(loss_fn))`.  The recomputation itself is the graph pass in
    alpa_b200/parallel/remat.py, run by the compile functions on the traced step."""
    def decorate(f):
        @functools.wraps(f)
        def wrapped(*args, **kwargs):
            from alpa_b200.parallel.remat import request_remat
            request_remat(True)
            return f(*args, **kwargs)
        return wrapped
    return decorate(fun) if fun is not None else decorate


def automatic_remat(fun: Optional[Callable] = None, *, static_argnums: Sequence[int] = (),
                    layer_num: Optional[int] = None, eps: float = 0.6, **unused):
    """Like manual_remat, with the layer boundaries chosen automatically: the heavy operators of `fun` are clustered
    into `layer_num` layers of balanced FLOPs (reference: automatic_remat, layer_construction.py:573)."""
    def decorate(f):
        inner = automatic_layer_construction(f, layer_num, eps) if layer_num and layer_num > 1 else f
        return manual_remat(inner)
    return decorate(fun) if fun is not None else decorate


def checkpoint_layer(fn: Callable, *args):
    """Rematerialise `fn(*args)` in the backward pass; traceable."""
    from torch.utils.checkpoint import checkpoint
    return checkpoint(fn, *args, use_reentrant=False)
