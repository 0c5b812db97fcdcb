"""Front-end tracing: a Python train/eval step -> one flat fx graph of core-ATen + alpa_b200 primitives.

Reference: alpa/util.py:868-903 (trace_jaxpr_with_micro_batch) and :335-365 (jaxpr_to_hlo).  The
H100-native front end is torch: the step function is executed once on fake tensors under
``make_fx``; ``alpa_b200.grad`` calls ``torch.autograd.grad`` *inside* the traced function so the
graph contains forward, backward and the optimizer update, exactly like the reference's jaxpr.
"""
from __future__ import annotations

from typing import Any, Callable, Dict, Sequence, Tuple

import torch
from torch import fx
from torch.fx.experimental.proxy_tensor import make_fx
from torch._subclasses.fake_tensor import FakeTensorMode

aten = torch.ops.aten

_DECOMP_CACHE = None


def _mean_decomp(x, dim=None, keepdim=False, *, dtype=None):
    dims = list(range(x.dim())) if dim is None or (isinstance(dim, (list, tuple)) and len(dim) == 0) else (
        [dim] if isinstance(dim, int) else list(dim))
    count = 1
    for d in dims:
        count *= x.shape[d]
    if dtype is not None:
        x = x.to(dtype)
    return torch.sum(x, dims, keepdim) / count


def _addmm_decomp(bias, a, b, *, beta=1, alpha=1):
    out = torch.mm(a, b)
    if alpha != 1:
        out = out * alpha
    if beta == 0:
        return out
    return out + (bias if beta == 1 else bias * beta)


def _batch_norm_train_decomp(x, weight, bias, running_mean, running_var, training, momentum, eps):
    """Training-mode batch norm as reductions + element-wise math, so that a batch-sharded input yields partial
    statistics + an all-reduce (synchronised BN -- what XLA's SPMD partitioner produces for the reference)
    instead of forcing the batch dim to be replicated.  Running statistics are updated with a `copy_` of the new
    value: onto a cloned buffer that is functionalised away (alpa_b200.torch front end), onto a graph input it stays
    an input mutation like in eager PyTorch."""
    if not training:
        return NotImplemented
    dims = [0] + list(range(2, x.dim()))
    n = x.numel() // x.shape[1]
    shape = [1, -1] + [1] * (x.dim() - 2)
    xf = x.float()
    mean = xf.sum(dims) / n
    xc = xf - mean.view(shape)
    var = (xc * xc).sum(dims) / n
    rstd = torch.rsqrt(var + eps)
    y = xc * rstd.view(shape)
    if weight is not None:
        y = y * weight.float().view(shape)
    if bias is not None:
        y = y + bias.float().view(shape)
    if running_mean is not None:
        running_mean.copy_(((1 - momentum) * running_mean.float() + momentum * mean).to(running_mean.dtype))
    if running_var is not None:
        unbiased = var * (n / max(n - 1, 1))
        running_var.copy_(((1 - momentum) * running_var.float() + momentum * unbiased).to(running_var.dtype))
    return y.to(x.dtype), mean, rstd


def decomposition_table() -> Dict[Any, Callable]:
    """core-ATen decompositions minus the ops that have first-class sharding rules."""
    global _DECOMP_CACHE
    if _DECOMP_CACHE is None:
        from torch._decomp import core_aten_decompositions
        table = dict(core_aten_decompositions())
        keep_whole = [aten.embedding_dense_backward.default, aten._softmax_backward_data.default,
                      aten._log_softmax_backward_data.default, aten.native_layer_norm.default,
                      aten._softmax.default, aten._log_softmax.default, aten.embedding.default,
                      aten.convolution_backward.default,
                      aten.max_pool2d_with_indices_backward.default, aten.avg_pool2d_backward.default,
                      aten._adaptive_avg_pool2d_backward.default, aten.slice_backward.default,
                      aten.select_backward.default, aten.upsample_nearest2d_backward.default,
                      aten.native_group_norm.default, aten.upsample_nearest2d.default,
                      # the fused attention ops are differentiated through their own backward ops, which consume
                      # the forward's logsumexp: the export-style math decomposition of the forward alone would
                      # hand them the attention matrix instead (silently wrong gradients)
                      aten._scaled_dot_product_flash_attention_for_cpu.default]
        for op in keep_whole:
            table.pop(op, None)
        # addmm/baddbmm are not multilinear in the bias: split so a sharded contraction is reduced
        # *before* the bias is added (the reference gets this for free: XLA has dot + add)
        table[aten.native_batch_norm.default] = _batch_norm_train_decomp
        table[aten.addmm.default] = _addmm_decomp
        table[aten.mean.dim] = _mean_decomp
        table[aten.mean.default] = lambda x, *, dtype=None: _mean_decomp(x, None, False, dtype=dtype)
        _DECOMP_CACHE = table
    return _DECOMP_CACHE


def make_fake_inputs(avals: Sequence[Tuple[Tuple[int, ...], torch.dtype, Any]], device=None):
    """Fake (shape/dtype/device only) inputs for tracing -- no real memory is touched.  The fake tensors
    live on the *target* device so tensor constants created by the traced code land there too."""
    device = torch.device(device) if device is not None else torch.device("cpu")
    mode = FakeTensorMode(allow_non_fake_inputs=True)
    with mode:
        return [torch.empty(shape, dtype=dtype, device=device) for (shape, dtype, _dev) in avals], mode


def trace_flat_function(flat_fn: Callable, avals: Sequence[Tuple[Tuple[int, ...], torch.dtype, Any]],
                        device=None, fake_factories: bool = False) -> fx.GraphModule:
    """Trace `flat_fn(*tensors) -> list of tensors` with fake tensors of the given avals.

    `fake_factories`: also run the function body under the fake mode, so tensors it creates from nothing
    (`torch.randn(shape)`, `torch.zeros(...)`: parameter initialisers) are fake too.  Without it a create-state function
    materialises every full-size parameter on the tracing device before the plan that shards it even exists
    (GPT-15B: 210 GB on each 180 GB GPU)."""
    inputs, mode = make_fake_inputs(avals, device)
    # oneDNN's fused RNN layer (what nn.LSTM dispatches to on CPU) is an opaque op with a workspace side output; with
    # it disabled the recurrence is traced as per-step linear / gate math that the planner can shard
    prev = torch._C._get_mkldnn_enabled()
    torch._C._set_mkldnn_enabled(False)
    try:
        import contextlib
        with (mode if fake_factories else contextlib.nullcontext()):
            gm = make_fx(flat_fn, decomposition_table=decomposition_table(), tracing_mode="real",
                         _allow_non_fake_inputs=True)(*inputs)
    finally:
        torch._C._set_mkldnn_enabled(prev)
    _normalize_squeeze(gm)
    _functionalize_intermediate_inplace(gm)
    _eliminate_dead_code(gm)
    gm.recompile()
    fuse_epilogues(gm)
    return gm


_VIEW_LIKE = None


def _view_like_ops():
    global _VIEW_LIKE
    if _VIEW_LIKE is None:
        _VIEW_LIKE = {aten.view.default, aten._unsafe_view.default, aten.reshape.default, aten.permute.default,
                      aten.transpose.int, aten.t.default, aten.alias.default, aten.detach.default, aten.expand.default,
                      aten.squeeze.dim, aten.squeeze.dims, aten.squeeze.default, aten.unsqueeze.default,
                      aten.slice.Tensor, aten.select.int, aten.as_strided.default, aten.unflatten.int,
                      aten.flatten.using_ints, aten.narrow.default, aten.split.Tensor, aten.split_with_sizes.default,
                      aten.unbind.int, aten.chunk.default}

    return _VIEW_LIKE


def _functionalize_intermediate_inplace(gm: fx.GraphModule) -> int:
    """Some autograd formulas (addcdiv, clamp, ...) build their result with in-place ATen ops on freshly created
    temporaries: `t = empty(); t.copy_(a); t.div_(b); use(t)`.  In the trace `use` reads the node `copy_` and relies on
    the later `div_` having mutated the same storage -- an aliasing contract a sharded / staged executor does not keep
    (operands may be re-laid-out copies, stages may sit on different meshes).  Rewrite in-place ops whose target is an
    intermediate value into their functional form and point every later reader at the new value.  Mutations of graph
    inputs (optimizer kernels, running statistics) are left alone."""
    _view_like_ops()

    def base_is_input(n: fx.Node) -> bool:
        while isinstance(n, fx.Node) and n.op == "call_function" and n.target in _VIEW_LIKE:
            n = n.args[0]
        return not (isinstance(n, fx.Node) and n.op == "call_function")

    order = {n: i for i, n in enumerate(gm.graph.nodes)}
    changed = 0

    def stale_views(base: fx.Node, at: int, ignore=()) -> bool:
        """Is there a view of `base`, taken before position `at`, that is still read afterwards?  Such a reader would
        see the mutation in eager mode but not the functional value."""
        for v in base.users:
            if v in ignore or not (v.op == "call_function" and v.target in _VIEW_LIKE) or order.get(v, at) >= at:
                continue
            if any(order.get(u, -1) > at for u in v.users) or stale_views(v, at):
                return True
        return False

    for node in list(gm.graph.nodes):
        if node.op != "call_function" or not isinstance(node.target, torch._ops.OpOverload):
            continue
        t = node.target
        if t.namespace != "aten" or not t._schema.is_mutable:
            continue
        name = t._schema.name.split("::")[-1]
        if not name.endswith("_") or not node.args or not isinstance(node.args[0], fx.Node):
            continue
        dst = node.args[0]
        packet = getattr(aten, name[:-1], None)
        func = getattr(packet, t._overloadname, None) if packet is not None else None
        if func is None or base_is_input(dst):
            continue                      # no functional twin, or a write into a graph input: keep the mutation
        at = order[node]
        is_view = dst.op == "call_function" and dst.target in _VIEW_LIKE
        if not is_view:
            if stale_views(dst, at):
                continue
            with gm.graph.inserting_before(node):
                new = gm.graph.call_function(func, node.args, dict(node.kwargs))
            new.meta = dict(node.meta)
            for u in list(dst.users):
                if u is not new and u is not node and order.get(u, -1) > at:
                    u.replace_input_with(dst, new)
            node.replace_all_uses_with(new)
            gm.graph.erase_node(node)
            order[new] = at
            changed += 1
            continue
        # a write through a one-level slice / select of an intermediate buffer (`buf[..., 1:] = x`, `buf[..., 0] = c`):
        # new_buf = slice_scatter / select_scatter(buf, f(view, ...)), later readers of buf see new_buf
        base = dst.args[0]
        if dst.target not in (aten.slice.Tensor, aten.select.int) or not isinstance(base, fx.Node) or \
                base.op != "call_function" or base.target in _VIEW_LIKE or stale_views(base, at, ignore=(dst,)):
            continue
        with gm.graph.inserting_before(node):
            new_view = gm.graph.call_function(func, node.args, dict(node.kwargs))
            new_view.meta = dict(node.meta)
            if dst.target == aten.slice.Tensor:
                a = list(dst.args[1:]) + [None] * 4
                dim, start, end, step = (a[0] if a[0] is not None else 0), a[1], a[2], (a[3] if a[3] is not None else 1)
                new_base = gm.graph.call_function(aten.slice_scatter.default, (base, new_view, dim, start, end, step))
            else:
                new_base = gm.graph.call_function(aten.select_scatter.default, (base, new_view, dst.args[1], dst.args[2]))
            new_base.meta = dict(base.meta)
        for u in list(base.users):
            if u not in (dst, new_base) and order.get(u, -1) > at:
                u.replace_input_with(base, new_base)
        for u in list(dst.users):
            if u not in (node, new_view) and order.get(u, -1) > at:
                u.replace_input_with(dst, new_view)
        node.replace_all_uses_with(new_view)
        gm.graph.erase_node(node)
        order[new_view] = at
        order[new_base] = at + 0.5
        changed += 1
    return changed


def _eliminate_dead_code(gm: fx.GraphModule) -> int:
    """Dead-code elimination that also drops in-place ops whose target storage nobody reads.  fx keeps every mutating
    node alive; a forward pass that is traced but unused (the heavy-op profiling run of automatic layer construction,
    metrics computed and dropped) then survives through its `x.add_(y)` temporaries and drags whole sub-graphs along.
    A mutation of an intermediate buffer is live only if that buffer -- or a view of it -- is read by live code."""
    _view_like_ops()
    nodes = list(gm.graph.nodes)

    def root_of(n: fx.Node) -> fx.Node:
        while isinstance(n, fx.Node) and n.op == "call_function" and n.target in _VIEW_LIKE and n.args and \
                isinstance(n.args[0], fx.Node):
            n = n.args[0]
        return n

    def mutates_intermediate(n: fx.Node) -> bool:
        if n.op != "call_function" or not isinstance(n.target, torch._ops.OpOverload) or n.target.namespace != "aten":
            return False
        if not n.target._schema.is_mutable or not n.args or not isinstance(n.args[0], fx.Node):
            return False
        return root_of(n.args[0]).op == "call_function"

    roots = [n for n in nodes if n.op == "output" or (_is_impure(n) and n.op == "call_function"
                                                      and not mutates_intermediate(n))]
    live: set = set()

    def mark(n):
        stack = [n]
        while stack:
            m = stack.pop()
            if m in live:
                continue
            live.add(m)
            stack.extend(m.all_input_nodes)
    for r in roots:
        mark(r)
    pending = [n for n in nodes if mutates_intermediate(n)]
    changed = True
    while changed and pending:
        changed = False
        for n in list(pending):
            root = root_of(n.args[0])
            # the mutated storage is observed if its root buffer or any view derived from it is live
            seen, stack, observed = set(), [root], False
            while stack and not observed:
                v = stack.pop()
                if v in seen:
                    continue
                seen.add(v)
                if v in live or any(u in live for u in v.users if u is not n):
                    observed = True
                    break
                stack.extend(u for u in v.users if u.op == "call_function" and u.target in _VIEW_LIKE)
            if observed or n in live:
                mark(n)
                pending.remove(n)
                changed = True
    removed = 0
    for n in reversed(nodes):          # `live` is closed under inputs, so the users of a dead node are dead and gone
        if n.op in ("call_function", "get_attr") and n not in live and not n.users:
            gm.graph.erase_node(n)
            removed += 1
    return removed


def _normalize_squeeze(gm: fx.GraphModule) -> int:
    """`squeeze` decides by the size it sees at run time; on a shard a dim of global size n can have local size 1.
    Pin every squeeze to the dims that are 1 in the GLOBAL shape (and drop the ones that are global no-ops)."""
    changed = 0
    for node in list(gm.graph.nodes):
        if node.op != "call_function" or node.target not in (aten.squeeze.default, aten.squeeze.dim, aten.squeeze.dims):
            continue
        x = node.args[0]
        v = x.meta.get("val") if isinstance(x, fx.Node) else None
        if not isinstance(v, torch.Tensor):
            continue
        nd = v.dim()
        if node.target == aten.squeeze.default:
            cand = list(range(nd))
        elif node.target == aten.squeeze.dim:
            cand = [int(node.args[1]) % nd] if nd else []
        else:
            cand = [int(d) % nd for d in node.args[1]] if nd else []
        dims = sorted({d for d in cand if int(v.shape[d]) == 1})
        if dims:
            if node.target == aten.squeeze.dims and list(node.args[1]) == dims:
                continue
            with gm.graph.inserting_before(node):
                new = gm.graph.call_function(aten.squeeze.dims, (x, dims))
            new.meta = dict(node.meta)
            node.replace_all_uses_with(new)
        else:
            node.replace_all_uses_with(x)
        gm.graph.erase_node(node)
        changed += 1
    return changed


def _is_impure(node: fx.Node) -> bool:
    if node.op in ("placeholder", "output"):
        return True
    if node.op == "call_function":
        t = node.target
        if t == torch.ops.alpa_b200.fused_adamw_.default:
            return True
        schema = getattr(t, "_schema", None)
        if schema is not None and schema.is_mutable:
            return True
    return False


# ------------------------------------------------------------------------------------------------
# graph-level kernel fusion (peephole): the XLA fusion passes of the reference have no counterpart
# here because the primitives already are fused kernels; what remains is stitching an element-wise
# backward into the epilogue of the GEMM that produces its input.
# ------------------------------------------------------------------------------------------------
def fuse_epilogues(gm: fx.GraphModule) -> int:
    """act_bwd(linear_dgrad(dy, w), z, act)  ->  linear_dgrad_act(dy, w, z, act)   (dGELU/dReLU in the
    dgrad GEMM epilogue: removes one read+write of the [tokens, 4H] gradient per MLP)."""
    ab = torch.ops.alpa_b200
    n_fused = 0
    for node in list(gm.graph.nodes):
        if node.op != "call_function" or node.target != ab.act_bwd.default:
            continue
        dy, z, act = node.args[0], node.args[1], node.args[2]
        if not (isinstance(dy, fx.Node) and dy.op == "call_function" and dy.target == ab.linear_dgrad.default):
            continue
        if len(dy.users) != 1 or act not in ("gelu", "relu"):
            continue
        with gm.graph.inserting_before(node):
            fused = gm.graph.call_function(ab.linear_dgrad_act.default, (dy.args[0], dy.args[1], z, act))
        fused.meta = dict(node.meta)
        node.replace_all_uses_with(fused)
        gm.graph.erase_node(node)
        gm.graph.erase_node(dy)
        n_fused += 1
    # add(linear_dgrad(dy, w), r) -> linear_dgrad_add(dy, w, r): gradient accumulation across the two consumers of an
    # activation (residual branch + linear) in the dgrad GEMM epilogue instead of a separate element-wise kernel
    aten = torch.ops.aten
    import os as _os
    # off by default: measured on GPT-1.3B (same box, profiles/r2_ab_*): the residual read makes the epilogue-bound
    # dgrad GEMMs 1.9 ms slower per step while the 48 separate add kernels cost 1.5 ms
    fuse_add = _os.environ.get("ALPA_B200_FUSE_DGRAD_ADD", "0") not in ("0", "false")
    for node in list(gm.graph.nodes):
        if not fuse_add:
            break
        if node.op != "call_function" or node.target != aten.add.Tensor or len(node.args) != 2:
            continue
        if node.kwargs.get("alpha", 1) != 1:
            continue
        a, b = node.args
        if not (isinstance(a, fx.Node) and isinstance(b, fx.Node)):
            continue
        for dg, other in ((a, b), (b, a)):
            if dg.op == "call_function" and dg.target == ab.linear_dgrad.default and len(dg.users) == 1:
                v1, v2, vo = dg.meta.get("val"), other.meta.get("val"), node.meta.get("val")
                if not all(isinstance(v, torch.Tensor) for v in (v1, v2, vo)):
                    continue
                if v1.shape != v2.shape or v1.dtype != v2.dtype or vo.dtype != v1.dtype:
                    continue
                with gm.graph.inserting_before(node):
                    fused = gm.graph.call_function(ab.linear_dgrad_add.default, (dg.args[0], dg.args[1], other))
                fused.meta = dict(node.meta)
                node.replace_all_uses_with(fused)
                gm.graph.erase_node(node)
                gm.graph.erase_node(dg)
                n_fused += 1
                break
    if n_fused:
        gm.graph.lint()
        gm.recompile()
    return n_fused
