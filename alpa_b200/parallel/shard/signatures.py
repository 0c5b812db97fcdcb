"""Sharding signatures of operators: the front end of the auto-sharding planner.

Every node of the traced graph (core-ATen ops + ``alpa_b200`` primitives) is described by an
einsum-like *label signature*: each dim of each tensor operand / output carries a label id; labels are
SHARDABLE or NOSHARD.  The native planner (``alpa_b200/csrc/auto_sharding.cpp``) turns signatures into
strategies: a strategy assigns logical-mesh axes to labels; a sharded label that is absent from an
output means that output is a partial sum and is all-reduced.  This replaces the reference's
per-HLO-opcode strategy registration (XLA/service/spmd/auto_sharding.cc:537-1439 and
auto_sharding_dot_handler.cc) with one declarative table.
"""
from __future__ import annotations

import math
import operator
from dataclasses import dataclass, field
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple

import torch
from torch import fx

aten = torch.ops.aten
SHARD, NOSHARD = 0, 1


@dataclass
class OpSig:
    labels: List[Tuple[int, int]] = field(default_factory=list)            # (size, kind)
    operands: List[Tuple[fx.Node, List[int]]] = field(default_factory=list)  # tensor operands, labels/dim
    outputs: List[Tuple[Tuple[int, ...], List[int], torch.dtype]] = field(default_factory=list)
    follow: int = -1
    flops: float = 0.0
    kind: str = "compute"          # compute | constant
    reduce_op: str = "sum"         # collective op for partial outputs
    # executor hook: (node, ctx) -> (args, kwargs) with local shapes / shard offsets substituted
    localize: Optional[Callable] = None
    # per output: indices of the operands it is computed from (None / missing = all); see planner.h Output.depends
    output_depends: Optional[List[List[int]]] = None
    zero_compatible: bool = False  # element-wise math that may run on a ZeRO shard
    # operands that are *added* to the (possibly partial) result, e.g. a bias: when the output is a
    # partial sum they are applied on one device of the reduction group only (others get None)
    additive_operands: List[int] = field(default_factory=list)
    # planner hints (None = derive from the op's schema): operand indices updated in place; whether outputs are new memory
    mutated: Optional[List[int]] = None
    allocates: Optional[bool] = None

    def new(self, size: int, kind: int = SHARD) -> int:
        self.labels.append((int(size), kind if size > 1 else NOSHARD))
        return len(self.labels) - 1


def _val(n):
    return n.meta.get("val") if isinstance(n, fx.Node) else None


def _is_tensor_node(n) -> bool:
    return isinstance(n, fx.Node) and isinstance(_val(n), torch.Tensor)


def _shape(n) -> Tuple[int, ...]:
    return tuple(int(s) for s in _val(n).shape)


def _out_vals(node) -> List[torch.Tensor]:
    v = _val(node)
    if isinstance(v, torch.Tensor):
        return [v]
    if isinstance(v, (list, tuple)):
        return [t for t in v if isinstance(t, torch.Tensor)]
    return []


def _numel(shape) -> int:
    return int(math.prod(shape)) if len(shape) else 1


def _choose_follow(sig: OpSig, prefer_shape: Optional[Tuple[int, ...]] = None) -> int:
    """Follow the largest operand, preferring one that has the output's shape and is an activation.
    Operands that share no shardable label with the op (scalars, fully broadcast) cannot be followed:
    the node then becomes a leader and enumerates its own strategies (e.g. `expand` of a scalar)."""
    best, best_key = -1, None
    for i, (n, labels) in enumerate(sig.operands):
        if not any(l >= 0 and sig.labels[l][1] == SHARD for l in labels):
            continue
        shp = _shape(n)
        key = (prefer_shape is not None and shp == tuple(prefer_shape), _numel(shp), n.op != "placeholder", -i)
        if best_key is None or key > best_key:
            best, best_key = i, key
    return best


# ------------------------------------------------------------------------------------------------
# generic rules
# ------------------------------------------------------------------------------------------------
def _tensor_args(node: fx.Node) -> List[fx.Node]:
    out = []

    def visit(a):
        if _is_tensor_node(a):
            out.append(a)
        elif isinstance(a, (list, tuple)):
            for x in a:
                visit(x)

    for a in node.args:
        visit(a)
    for a in node.kwargs.values():
        visit(a)
    return out


def rule_pointwise(node: fx.Node) -> OpSig:
    sig = OpSig()
    outs = _out_vals(node)
    oshape = tuple(int(s) for s in outs[0].shape)
    olabels = [sig.new(s) for s in oshape]
    for a in _tensor_args(node):
        shp = _shape(a)
        labels = []
        off = len(oshape) - len(shp)
        for d, s in enumerate(shp):
            od = d + off
            labels.append(olabels[od] if (od >= 0 and s == oshape[od] and s > 1) else -1)
        sig.operands.append((a, labels))
    for o in outs:
        sig.outputs.append((tuple(int(s) for s in o.shape), list(olabels), o.dtype))
    if sig.operands:
        sig.follow = _choose_follow(sig, oshape)
    else:
        sig.kind = "constant"
    sig.zero_compatible = True
    return sig


def rule_replicated(node: fx.Node) -> OpSig:
    """Fallback: nothing is shardable -> the op runs replicated on gathered operands."""
    sig = OpSig()
    for a in _tensor_args(node):
        sig.operands.append((a, [sig.new(s, NOSHARD) for s in _shape(a)]))
    for o in _out_vals(node):
        sig.outputs.append((tuple(int(s) for s in o.shape), [sig.new(s, NOSHARD) for s in o.shape], o.dtype))
    if sig.operands:
        sig.follow = _choose_follow(sig)
    else:
        sig.kind = "constant"
    return sig


def _dimwise(node: fx.Node, x: fx.Node, noshard_dims: Sequence[int], out_map: Optional[Dict[int, int]] = None,
             extra_operands: Sequence[Tuple[fx.Node, Dict[int, int]]] = ()) -> OpSig:
    """Ops that act independently along all dims of `x` except `noshard_dims`.
    out_map: output dim -> input dim (None = same rank identity).  extra_operands: (node, {dim: x dim})."""
    sig = OpSig()
    shp = _shape(x)
    nd = len(shp)
    ns = {d % nd for d in noshard_dims} if nd else set()
    xl = [sig.new(s, NOSHARD if d in ns else SHARD) for d, s in enumerate(shp)]
    sig.operands.append((x, xl))
    for (n, dm) in extra_operands:
        labels = []
        for d, s in enumerate(_shape(n)):
            xd = dm.get(d)
            labels.append(xl[xd] if (xd is not None and s == shp[xd] and s > 1) else (sig.new(s, NOSHARD) if s > 1 else -1))
        sig.operands.append((n, labels))
    for o in _out_vals(node):
        oshape = tuple(int(s) for s in o.shape)
        if out_map is None:
            ol = [xl[d] if (d < nd and oshape[d] == shp[d] and d not in ns) else sig.new(oshape[d], NOSHARD)
                  for d in range(len(oshape))]
        else:
            ol = []
            for d in range(len(oshape)):
                xd = out_map.get(d)
                ol.append(xl[xd] if (xd is not None and oshape[d] == shp[xd] and xd not in ns)
                          else sig.new(oshape[d], NOSHARD))
        sig.outputs.append((oshape, ol, o.dtype))
    sig.follow = _choose_follow_fixed(sig, 0)
    return sig


def _choose_follow_fixed(sig: OpSig, idx: int) -> int:
    """`idx` if that operand can be followed, else the best alternative (or leader)."""
    if idx < len(sig.operands):
        labels = sig.operands[idx][1]
        if any(l >= 0 and sig.labels[l][1] == SHARD for l in labels):
            return idx
    return _choose_follow(sig)


def rule_permute(node: fx.Node) -> OpSig:
    x = node.args[0]
    nd = len(_shape(x))
    if node.target in (aten.t.default,):
        perm = [1, 0] if nd == 2 else list(range(nd))
    elif node.target in (aten.transpose.int,):
        d0, d1 = node.args[1] % nd, node.args[2] % nd
        perm = list(range(nd))
        perm[d0], perm[d1] = perm[d1], perm[d0]
    else:
        perm = [p % nd for p in node.args[1]]
    sig = OpSig()
    xl = [sig.new(s) for s in _shape(x)]
    sig.operands.append((x, xl))
    o = _out_vals(node)[0]
    sig.outputs.append((tuple(int(s) for s in o.shape), [xl[p] for p in perm], o.dtype))
    sig.follow = 0
    sig.zero_compatible = True
    return sig


def reshape_dim_groups(in_shape: Sequence[int], out_shape: Sequence[int]):
    """Pair up (in_dim, out_dim) whose *major* factor coincides so a tiling of one maps to a tiling of
    the other.  Returns list of (in_dim, out_dim, shardable_size)."""
    pairs = []
    i = j = 0
    ni, no = len(in_shape), len(out_shape)
    while i < ni and j < no:
        if in_shape[i] == 1:
            i += 1
            continue
        if out_shape[j] == 1:
            j += 1
            continue
        # start of a group: dims i.. and j.. whose products match
        pi, pj = in_shape[i], out_shape[j]
        i0, j0 = i, j
        while pi != pj:
            if pi < pj:
                i += 1
                if i >= ni:
                    return pairs
                pi *= in_shape[i]
            else:
                j += 1
                if j >= no:
                    return pairs
                pj *= out_shape[j]
        pairs.append((i0, j0, min(in_shape[i0], out_shape[j0])))
        i += 1
        j += 1
    return pairs


def rule_reshape(node: fx.Node) -> OpSig:
    x = node.args[0]
    ishape = _shape(x)
    o = _out_vals(node)[0]
    oshape = tuple(int(s) for s in o.shape)
    sig = OpSig()
    il: List[int] = [-2] * len(ishape)
    ol: List[int] = [-2] * len(oshape)
    for (i, j, size) in reshape_dim_groups(ishape, oshape):
        l = sig.new(size)
        il[i] = l
        ol[j] = l
    for d, s in enumerate(ishape):
        if il[d] == -2:
            il[d] = sig.new(s, NOSHARD) if s > 1 else -1
    for d, s in enumerate(oshape):
        if ol[d] == -2:
            ol[d] = sig.new(s, NOSHARD) if s > 1 else -1
    sig.operands.append((x, il))
    sig.outputs.append((oshape, ol, o.dtype))
    sig.follow = 0
    sig.zero_compatible = True

    def localize(node, ctx):
        args = list(node.args)
        args[1] = list(ctx.local_out_shape(0))
        return tuple(args), dict(node.kwargs)

    if node.target in (aten.view.default, aten._unsafe_view.default, aten.reshape.default):
        sig.localize = localize
    return sig


def rule_expand(node: fx.Node) -> OpSig:
    x = node.args[0]
    ishape = _shape(x)
    o = _out_vals(node)[0]
    oshape = tuple(int(s) for s in o.shape)
    sig = OpSig()
    ol = [sig.new(s) for s in oshape]
    off = len(oshape) - len(ishape)
    il = [ol[d + off] if (s == oshape[d + off] and s > 1) else -1 for d, s in enumerate(ishape)]
    sig.operands.append((x, il))
    sig.outputs.append((oshape, ol, o.dtype))
    sig.follow = 0

    def localize(node, ctx):
        args = list(node.args)
        args[1] = list(ctx.local_out_shape(0))
        return tuple(args), dict(node.kwargs)

    sig.localize = localize
    return sig


def _norm_dims(dims, nd):
    if dims is None or (isinstance(dims, (list, tuple)) and len(dims) == 0):
        return list(range(nd))
    if isinstance(dims, int):
        dims = [dims]
    return sorted({d % nd for d in dims}) if nd else []


def rule_reduce(node: fx.Node, reduce_op="sum") -> OpSig:
    x = node.args[0]
    ishape = _shape(x)
    nd = len(ishape)
    dims = node.args[1] if len(node.args) > 1 and not isinstance(node.args[1], bool) else None
    if node.target in (aten.sum.default, aten.max.default, aten.min.default):
        dims = None
    rd = set(_norm_dims(dims, nd))
    sig = OpSig(reduce_op=reduce_op)
    il = [sig.new(s) for s in ishape]
    sig.operands.append((x, il))
    for o in _out_vals(node):
        oshape = tuple(int(s) for s in o.shape)
        keep = len(oshape) == nd
        ol = []
        k = 0
        for d in range(nd):
            if d in rd:
                if keep:
                    ol.append(-1)
            else:
                ol.append(il[d])
            k += 1
        sig.outputs.append((oshape, ol, o.dtype))
    sig.follow = 0
    sig.flops = 0
    return sig


def rule_mm(node: fx.Node) -> OpSig:
    sig = OpSig()
    o = _out_vals(node)[0]
    if node.target == aten.addmm.default:
        bias, a, b = node.args[0], node.args[1], node.args[2]
    else:
        bias, (a, b) = None, node.args[:2]
    ash, bsh = _shape(a), _shape(b)
    if len(ash) == 3:  # bmm
        lb, lm, lk, ln = sig.new(ash[0]), sig.new(ash[1]), sig.new(ash[2]), sig.new(bsh[2])
        sig.operands += [(a, [lb, lm, lk]), (b, [lb, lk, ln])]
        ol = [lb, lm, ln]
        sig.flops = 2.0 * ash[0] * ash[1] * ash[2] * bsh[2]
    else:
        lm, lk, ln = sig.new(ash[0]), sig.new(ash[1]), sig.new(bsh[1])
        sig.operands += [(a, [lm, lk]), (b, [lk, ln])]
        ol = [lm, ln]
        sig.flops = 2.0 * ash[0] * ash[1] * bsh[1]
    if bias is not None and _is_tensor_node(bias):
        bshp = _shape(bias)
        off = len(ol) - len(bshp)
        sig.operands.insert(0, (bias, [ol[d + off] if s == o.shape[d + off] and s > 1 else -1 for d, s in enumerate(bshp)]))
    sig.outputs.append((tuple(int(s) for s in o.shape), ol, o.dtype))
    return sig


def rule_softmax(node: fx.Node) -> OpSig:
    return _dimwise(node, node.args[0], [node.args[1]])


def rule_native_layer_norm(node: fx.Node) -> OpSig:
    x, nshape, w, b = node.args[0], node.args[1], node.args[2], node.args[3]
    nd = len(_shape(x))
    k = len(nshape)
    ns = list(range(nd - k, nd))
    extra = []
    for p in (w, b):
        if _is_tensor_node(p):
            extra.append((p, {}))
    return _dimwise(node, x, ns, extra_operands=extra)


def rule_embedding(node: fx.Node) -> OpSig:
    w, ids = node.args[0], node.args[1]
    sig = OpSig()
    lv = sig.new(_shape(w)[0], NOSHARD)  # plain aten.embedding: keep the table rows whole
    lh = sig.new(_shape(w)[1])
    idl = [sig.new(s) for s in _shape(ids)]
    sig.operands += [(w, [lv, lh]), (ids, idl)]
    o = _out_vals(node)[0]
    sig.outputs.append((tuple(int(s) for s in o.shape), idl + [lh], o.dtype))
    sig.follow = 1
    return sig


def rule_embedding_dense_backward(node: fx.Node) -> OpSig:
    g, ids = node.args[0], node.args[1]
    sig = OpSig()
    idl = [sig.new(s) for s in _shape(ids)]
    lh = sig.new(_shape(g)[-1])
    sig.operands += [(g, idl + [lh]), (ids, idl)]
    o = _out_vals(node)[0]
    sig.outputs.append((tuple(int(s) for s in o.shape), [sig.new(o.shape[0], NOSHARD), lh], o.dtype))
    sig.follow = 0
    return sig


def rule_dim_op(dim_arg_index: int, x_index: int = 0, extra: Sequence[int] = (), default_dim=0):
    """Ops that work along `dim` (an int, a list of ints, or None = all dims): that dim stays whole, the others are
    element-wise.  `dim_arg_index` is the positional index of the dim argument in the op's schema."""
    def rule(node: fx.Node) -> OpSig:
        x = node.args[x_index]
        dim = node.args[dim_arg_index] if len(node.args) > dim_arg_index else node.kwargs.get(
            "dim", node.kwargs.get("dims", default_dim))
        nd = len(_shape(x))
        if dim is None or (isinstance(dim, (list, tuple)) and len(dim) == 0):
            dims = list(range(nd))                      # flattened semantics (argmax(x), roll without dims)
        elif isinstance(dim, (list, tuple)):
            dims = [int(d) for d in dim]
        else:
            dims = [int(dim)]
        ex = []
        for i in extra:
            if len(node.args) > i and _is_tensor_node(node.args[i]):
                n = node.args[i]
                ex.append((n, {d: d for d in range(len(_shape(n)))} if len(_shape(n)) == nd else {}))
        return _dimwise(node, x, dims, extra_operands=ex)
    return rule


def rule_select(node: fx.Node) -> OpSig:
    x, dim = node.args[0], node.args[1]
    nd = len(_shape(x))
    dim %= nd
    out_map = {}
    k = 0
    for d in range(nd):
        if d == dim:
            continue
        out_map[k] = d
        k += 1
    return _dimwise(node, x, [dim], out_map=out_map)


def rule_cat(node: fx.Node) -> OpSig:
    tensors = node.args[0]
    dim = node.args[1] if len(node.args) > 1 else 0
    sig = OpSig()
    o = _out_vals(node)[0]
    oshape = tuple(int(s) for s in o.shape)
    dim %= len(oshape)
    ol = [sig.new(s, NOSHARD if d == dim else SHARD) for d, s in enumerate(oshape)]
    for t in tensors:
        sig.operands.append((t, [ol[d] if d != dim else sig.new(s, NOSHARD) for d, s in enumerate(_shape(t))]))
    sig.outputs.append((oshape, ol, o.dtype))
    sig.follow = _choose_follow(sig)
    return sig


def rule_constant(node: fx.Node) -> OpSig:
    sig = OpSig(kind="constant")
    for o in _out_vals(node):
        sig.outputs.append((tuple(int(s) for s in o.shape), [sig.new(s) for s in o.shape], o.dtype))

    def localize(node, ctx):
        args = list(node.args)
        if args and isinstance(args[0], (list, tuple)):
            args[0] = list(ctx.local_out_shape(0))
        return tuple(args), dict(node.kwargs)

    if node.target in (aten.full.default, aten.zeros.default, aten.ones.default, aten.empty.memory_format,
                       aten.rand.default, aten.randn.default):
        sig.localize = localize
    else:  # arange / scalar_tensor etc: never sharded
        sig.labels = [(s, NOSHARD) for (s, _) in sig.labels]
    return sig


def rule_getitem(node: fx.Node) -> OpSig:
    src, idx = node.args
    sig = OpSig()
    o = _out_vals(node)[0]
    labels = [sig.new(s) for s in o.shape]
    sig.operands.append((src, labels))
    sig.outputs.append((tuple(int(s) for s in o.shape), labels, o.dtype))
    sig.follow = 0
    sig.zero_compatible = True
    return sig


def rule_convolution(node: fx.Node) -> OpSig:
    """convolution(x [N,Ci,*], w, bias, stride, padding, dilation, transposed, output_padding, groups).
    Weight layout: [Co, Ci/groups, *k], or [Ci, Co/groups, *k] for transposed convolutions."""
    x, w, b = node.args[0], node.args[1], node.args[2]
    sig = OpSig()
    xs, ws = _shape(x), _shape(w)
    transposed = bool(node.args[6]) if len(node.args) > 6 else False
    groups = node.args[8] if len(node.args) > 8 else 1
    o = _out_vals(node)[0]
    kind = SHARD if groups == 1 else NOSHARD
    ln = sig.new(xs[0])
    lci = sig.new(xs[1], kind)
    lco = sig.new(int(o.shape[1]), kind)
    sp_in = [sig.new(s, NOSHARD) for s in xs[2:]]
    sp_k = [sig.new(s, NOSHARD) for s in ws[2:]]
    sp_out = [sig.new(s, NOSHARD) for s in o.shape[2:]]
    if groups == 1:
        wl = [lci, lco] if transposed else [lco, lci]
    else:
        wl = [sig.new(ws[0], NOSHARD), sig.new(ws[1], NOSHARD)]
    sig.operands += [(x, [ln, lci] + sp_in), (w, wl + sp_k)]
    if _is_tensor_node(b):
        sig.operands.append((b, [lco]))
        sig.additive_operands.append(2)      # input channels sharded -> partial sums: add the bias once
    sig.outputs.append((tuple(int(s) for s in o.shape), [ln, lco] + sp_out, o.dtype))
    sig.flops = 2.0 * _numel(o.shape) * (ws[0] if transposed else ws[1]) * _numel(ws[2:])
    return sig


def rule_convolution_backward(node: fx.Node) -> OpSig:
    """convolution_backward(grad_out, input, weight, bias_sizes, stride, padding, dilation, transposed, output_padding,
    groups, output_mask) -> (grad_input, grad_weight, grad_bias)"""
    g, x, w = node.args[0], node.args[1], node.args[2]
    sig = OpSig()
    xs, ws, gs = _shape(x), _shape(w), _shape(g)
    transposed = bool(node.args[7]) if len(node.args) > 7 else False
    groups = node.args[9] if len(node.args) > 9 else 1
    kind = SHARD if groups == 1 else NOSHARD
    ln, lci, lco = sig.new(xs[0]), sig.new(xs[1], kind), sig.new(gs[1], kind)
    sp_in = [sig.new(s, NOSHARD) for s in xs[2:]]
    sp_k = [sig.new(s, NOSHARD) for s in ws[2:]]
    sp_g = [sig.new(s, NOSHARD) for s in gs[2:]]
    if groups == 1:
        wl = [lci, lco] if transposed else [lco, lci]
    else:
        wl = [sig.new(ws[0], NOSHARD), sig.new(ws[1], NOSHARD)]
    sig.operands += [(g, [ln, lco] + sp_g), (x, [ln, lci] + sp_in), (w, wl + sp_k)]
    v = _val(node)
    # grad_input = f(grad_out, weight), grad_weight = f(grad_out, input), grad_bias = f(grad_out)
    outs = [(0, [ln, lci] + sp_in, [0, 2]), (1, wl + sp_k, [0, 1]), (2, [lco], [0])]
    sig.output_depends = []
    for i, labels, deps in outs:
        t = v[i]
        if isinstance(t, torch.Tensor):
            sig.outputs.append((tuple(int(s) for s in t.shape), labels, t.dtype))
            sig.output_depends.append(deps)
    sig.flops = 4.0 * _numel(gs) * (ws[0] if transposed else ws[1]) * _numel(ws[2:])
    return sig


def rule_pool(node: fx.Node) -> OpSig:
    x = node.args[0]
    nd = len(_shape(x))
    extra = [(a, {d: d for d in range(len(_shape(a)))}) for a in node.args[1:]
             if _is_tensor_node(a) and len(_shape(a)) == nd]
    sig = _dimwise(node, x, list(range(2, nd)), extra_operands=extra)
    if node.target == aten.upsample_nearest2d_backward.default:
        def localize(node, ctx):     # (grad_output, output_size, input_size, ...): input_size is the result's shape
            args = list(node.args)
            args[2] = list(ctx.local_out_shape(0))
            return tuple(args), dict(node.kwargs)
        sig.localize = localize
    return sig


def rule_constant_pad(node: fx.Node) -> OpSig:
    """constant_pad_nd(x, pad): padded dims stay whole, the others are element-wise."""
    x, pad = node.args[0], node.args[1]
    nd = len(_shape(x))
    padded = [nd - 1 - i for i in range(len(pad) // 2) if pad[2 * i] != 0 or pad[2 * i + 1] != 0]
    return _dimwise(node, x, padded)


def rule_batch_norm(node: fx.Node) -> OpSig:
    # statistics are computed over (N, spatial): keep those whole, shard channels only
    x = node.args[0]
    nd = len(_shape(x))
    extra = [(a, {0: 1}) for a in node.args[1:5] if _is_tensor_node(a)]
    sig = _dimwise(node, x, [0] + list(range(2, nd)), extra_operands=extra)
    # outputs 1.. are per-channel vectors
    xl = sig.operands[0][1]
    fixed = []
    for (shape, labels, dt) in sig.outputs:
        if len(shape) == 1 and shape[0] == _shape(x)[1]:
            labels = [xl[1]]
        fixed.append((shape, labels, dt))
    sig.outputs = fixed
    return sig


def rule_group_norm(node: fx.Node) -> OpSig:
    """native_group_norm(x [N,C,*], weight, bias, N, C, HxW, groups, eps) -> (y, mean [N,G], rstd [N,G]):
    statistics are per sample, so the batch dim is shardable (N argument localised); channels are not."""
    x = node.args[0]
    xs = _shape(x)
    sig = OpSig()
    ln, lc = sig.new(xs[0]), sig.new(xs[1], NOSHARD)
    sp = [sig.new(s, NOSHARD) for s in xs[2:]]
    sig.operands.append((x, [ln, lc] + sp))
    for a in node.args[1:3]:
        if _is_tensor_node(a):
            sig.operands.append((a, [lc]))
    outs = _out_vals(node)
    sig.outputs.append((tuple(int(d) for d in outs[0].shape), [ln, lc] + sp, outs[0].dtype))
    for o in outs[1:]:
        lg = sig.new(int(o.shape[1]), NOSHARD)
        sig.outputs.append((tuple(int(d) for d in o.shape), [ln, lg], o.dtype))
    sig.named = {"batch": ln}
    sig.follow = 0

    def localize(node, ctx):
        args = list(node.args)
        args[3] = ctx.local_size("batch")
        return tuple(args), dict(node.kwargs)
    sig.localize = localize
    return sig


# ------------------------------------------------------------------------------------------------
# alpa_b200 primitives
# ------------------------------------------------------------------------------------------------
def _lead_labels(sig: OpSig, shape: Sequence[int]) -> List[int]:
    return [sig.new(s) for s in shape]


def rule_ab_linear(node: fx.Node) -> OpSig:
    x, w = node.args[0], node.args[1]
    b = node.args[2] if len(node.args) > 2 else None
    sig = OpSig()
    xs, ws = _shape(x), _shape(w)
    lead = _lead_labels(sig, xs[:-1])
    has_act = node.target == torch.ops.alpa_b200.linear_act.default and node.args[3] != "none"
    # a non-linear epilogue forbids splitting the contraction (act(sum) != sum(act))
    lk, ln = sig.new(xs[-1], NOSHARD if has_act else SHARD), sig.new(ws[0])
    sig.operands += [(x, lead + [lk]), (w, [ln, lk])]
    if _is_tensor_node(b):
        sig.operands.append((b, [ln]))
        sig.additive_operands.append(len(sig.operands) - 1)
    for o in _out_vals(node):
        sig.outputs.append((tuple(int(s) for s in o.shape), lead + [ln], o.dtype))
    sig.flops = 2.0 * _numel(xs) * ws[0]
    return sig


def rule_ab_linear_dgrad(node: fx.Node) -> OpSig:
    dy, w = node.args[0], node.args[1]
    sig = OpSig()
    ds, ws = _shape(dy), _shape(w)
    lead = _lead_labels(sig, ds[:-1])
    ln, lk = sig.new(ds[-1]), sig.new(ws[1])
    sig.operands += [(dy, lead + [ln]), (w, [ln, lk])]
    if len(node.args) > 2 and _is_tensor_node(node.args[2]):  # fused act backward / fused accumulation: dx's layout
        sig.operands.append((node.args[2], lead + [lk]))
        if node.target == torch.ops.alpa_b200.linear_dgrad_add.default:
            sig.additive_operands = [2]      # added once: on one device of the group when dx is a partial sum
    o = _out_vals(node)[0]
    sig.outputs.append((tuple(int(s) for s in o.shape), lead + [lk], o.dtype))
    sig.flops = 2.0 * _numel(ds) * ws[1]
    return sig


def rule_ab_linear_wgrad(node: fx.Node) -> OpSig:
    dy, x = node.args[0], node.args[1]
    sig = OpSig()
    ds, xs = _shape(dy), _shape(x)
    lead = _lead_labels(sig, ds[:-1])
    ln, lk = sig.new(ds[-1]), sig.new(xs[-1])
    sig.operands += [(dy, lead + [ln]), (x, lead + [lk])]
    o = _out_vals(node)[0]
    sig.outputs.append((tuple(int(s) for s in o.shape), [ln, lk], o.dtype))
    sig.flops = 2.0 * _numel(ds) * xs[-1]
    return sig


def rule_ab_bias_grad(node: fx.Node) -> OpSig:
    dy = node.args[0]
    sig = OpSig()
    ds = _shape(dy)
    lead = _lead_labels(sig, ds[:-1])
    ln = sig.new(ds[-1])
    sig.operands.append((dy, lead + [ln]))
    o = _out_vals(node)[0]
    sig.outputs.append((tuple(int(s) for s in o.shape), [ln], o.dtype))
    sig.follow = 0
    return sig


def rule_ab_layer_norm(node: fx.Node) -> OpSig:
    """layer_norm(x,g,b,eps) / add_layer_norm(x,r,g,b,eps) and their RMS forms rms_norm(x,g,eps) /
    add_rms_norm(x,r,g,eps): rows shard, the normalised dim never does"""
    is_add = node.target in (torch.ops.alpa_b200.add_layer_norm.default, torch.ops.alpa_b200.add_rms_norm.default)
    x = node.args[0]
    sig = OpSig()
    xs = _shape(x)
    lead = _lead_labels(sig, xs[:-1])
    lh = sig.new(xs[-1], NOSHARD)
    sig.operands.append((x, lead + [lh]))
    rest = node.args[1:]
    if is_add:
        sig.operands.append((rest[0], lead + [lh]))
        rest = rest[1:]
    for p in rest[:2]:
        if _is_tensor_node(p):
            sig.operands.append((p, [lh]))
    for o in _out_vals(node):
        oshape = tuple(int(s) for s in o.shape)
        sig.outputs.append((oshape, lead + [lh] if len(oshape) == len(xs) else list(lead), o.dtype))
    sig.follow = 0
    return sig


def rule_ab_layer_norm_bwd(node: fx.Node) -> OpSig:
    """layer_norm_bwd(dy,x,g,mean,rstd,dres) -> (dx,dgamma,dbeta) / rms_norm_bwd(dy,x,g,rstd,dres) -> (dx,dgamma)"""
    if node.target == torch.ops.alpa_b200.rms_norm_bwd.default:
        dy, x, g, rstd, dres = node.args[:5]
        stats = [rstd]
    else:
        dy, x, g, mean, rstd, dres = node.args[:6]
        stats = [mean, rstd]
    sig = OpSig()
    xs = _shape(x)
    lead = _lead_labels(sig, xs[:-1])
    lh = sig.new(xs[-1], NOSHARD)
    sig.operands += [(dy, lead + [lh]), (x, lead + [lh]), (g, [lh])] + [(t, list(lead)) for t in stats]
    if _is_tensor_node(dres):
        sig.operands.append((dres, lead + [lh]))
    v = _val(node)
    sig.outputs.append((tuple(int(s) for s in v[0].shape), lead + [lh], v[0].dtype))
    for t in v[1:]:   # dgamma (and dbeta): partial over rows
        sig.outputs.append((tuple(int(s) for s in t.shape), [lh], t.dtype))
    sig.follow = 0
    return sig


def rule_ab_attention(node: fx.Node) -> OpSig:
    q, k, v = node.args[:3]
    sig = OpSig()
    B, Sq, H, D = _shape(q)
    Sk = _shape(k)[1]
    lb, lh = sig.new(B), sig.new(H)
    lsq, lsk, ld = sig.new(Sq, NOSHARD), sig.new(Sk, NOSHARD), sig.new(D, NOSHARD)
    sig.operands += [(q, [lb, lsq, lh, ld]), (k, [lb, lsk, lh, ld]), (v, [lb, lsk, lh, ld])]
    vals = _val(node)
    sig.outputs.append((tuple(int(s) for s in vals[0].shape), [lb, lsq, lh, ld], vals[0].dtype))
    sig.outputs.append((tuple(int(s) for s in vals[1].shape), [lb, lh, lsq], vals[1].dtype))
    sig.follow = 0
    sig.flops = 4.0 * B * H * Sq * Sk * D
    return sig


def rule_ab_attention_cached(node: fx.Node) -> OpSig:
    """attention_cached(q, k_new, v_new, k_cache, v_cache, cache_len, scale) -> (o, k_cache', v_cache'): independent per
    (batch, head); the cache rows and the new block are never split (the append is a dynamic slice update)."""
    q, k_new, v_new, k_cache, v_cache, cache_len = node.args[:6]
    sig = OpSig()
    B, T, H, D = _shape(q)
    Sm = _shape(k_cache)[1]
    lb, lh = sig.new(B), sig.new(H)
    lt, ls, ld = sig.new(T, NOSHARD), sig.new(Sm, NOSHARD), sig.new(D, NOSHARD)
    new, cache = [lb, lt, lh, ld], [lb, ls, lh, ld]
    sig.operands += [(q, new), (k_new, new), (v_new, new), (k_cache, cache), (v_cache, cache)]
    if _is_tensor_node(cache_len):
        sig.operands.append((cache_len, [sig.new(1, NOSHARD) for _ in _shape(cache_len)]))
    vals = _val(node)
    for t, l in zip(vals, (new, cache, cache)):
        sig.outputs.append((tuple(int(s) for s in t.shape), list(l), t.dtype))
    sig.follow = 3            # the cache is the big operand: its layout decides (never move a cache to fit a token)
    sig.flops = 4.0 * B * H * T * Sm * D
    return sig


def rule_ab_attention_bwd(node: fx.Node) -> OpSig:
    do, q, k, v, o, lse = node.args[:6]
    sig = OpSig()
    B, Sq, H, D = _shape(q)
    Sk = _shape(k)[1]
    lb, lh = sig.new(B), sig.new(H)
    lsq, lsk, ld = sig.new(Sq, NOSHARD), sig.new(Sk, NOSHARD), sig.new(D, NOSHARD)
    qs, ks = [lb, lsq, lh, ld], [lb, lsk, lh, ld]
    sig.operands += [(do, qs), (q, qs), (k, ks), (v, ks), (o, qs), (lse, [lb, lh, lsq])]
    vals = _val(node)
    for t, l in zip(vals, (qs, ks, ks)):
        sig.outputs.append((tuple(int(s) for s in t.shape), list(l), t.dtype))
    sig.follow = 1
    sig.flops = 10.0 * B * H * Sq * Sk * D
    return sig


def rule_ab_attention_gqa_packed(node: fx.Node) -> OpSig:
    """attention_gqa_packed(qkv[B,S,Hkv,G+2,D]) / attention_gqa_packed_bwd(do, qkv, o, lse): batch and K/V heads
    shard; the slots of one K/V head (its G query heads, K and V) stay together, so a group is never split."""
    is_bwd = node.target == torch.ops.alpa_b200.attention_gqa_packed_bwd.default
    qkv = node.args[1] if is_bwd else node.args[0]
    sig = OpSig()
    B, S_, Hkv, P, D = _shape(qkv)
    G = P - 2
    lb, lkv = sig.new(B), sig.new(Hkv)
    ls, lslot, lg, ld = sig.new(S_, NOSHARD), sig.new(P, NOSHARD), sig.new(G, NOSHARD), sig.new(D, NOSHARD)
    packed, act, stat = [lb, ls, lkv, lslot, ld], [lb, ls, lkv, lg, ld], [lb, lkv, lg, ls]
    if is_bwd:
        do, _, o, lse = node.args[:4]
        sig.operands += [(do, act), (qkv, packed), (o, act), (lse, stat)]
        t = _out_vals(node)[0]
        sig.outputs.append((tuple(int(s) for s in t.shape), list(packed), t.dtype))
        sig.follow = 1
        sig.flops = 10.0 * B * Hkv * G * S_ * S_ * D
    else:
        sig.operands.append((qkv, packed))
        vals = _val(node)
        sig.outputs.append((tuple(int(s) for s in vals[0].shape), list(act), vals[0].dtype))
        sig.outputs.append((tuple(int(s) for s in vals[1].shape), list(stat), vals[1].dtype))
        sig.follow = 0
        sig.flops = 4.0 * B * Hkv * G * S_ * S_ * D
    return sig


def rule_ab_rotary_packed(node: fx.Node) -> OpSig:
    """rotary_packed(qkv[B,S,Hkv,G+2,D], position_ids[B,S], theta, inverse): batch and K/V heads shard; the slot dim and
    D (whose halves pair up) never do, and position_ids shares the batch and sequence labels (none on a broadcast
    batch dim: HF's [1, S])."""
    qkv, pos = node.args[:2]
    sig = OpSig()
    B, S_, Hkv, P, D = _shape(qkv)
    lb, ls, lkv = sig.new(B), sig.new(S_, NOSHARD), sig.new(Hkv)
    labels = [lb, ls, lkv, sig.new(P, NOSHARD), sig.new(D, NOSHARD)]
    pos_b = _shape(pos)[0]
    sig.operands += [(qkv, labels), (pos, [lb if pos_b == B else -1, ls])]
    t = _out_vals(node)[0]
    sig.outputs.append((tuple(int(s) for s in t.shape), list(labels), t.dtype))
    sig.follow = 0
    return sig


def rule_ab_swiglu(node: fx.Node) -> OpSig:
    """swiglu(gu[...,I,2]) -> h[...,I] / swiglu_bwd(dh[...,I], gu) -> dgu: the leading dims and I shard, the
    (gate, up) pair dim never does."""
    is_bwd = node.target == torch.ops.alpa_b200.swiglu_bwd.default
    gu = node.args[1] if is_bwd else node.args[0]
    sig = OpSig()
    gs = _shape(gu)
    lead = _lead_labels(sig, gs[:-1])
    pair = lead + [sig.new(gs[-1], NOSHARD)]
    if is_bwd:
        sig.operands += [(node.args[0], list(lead)), (gu, pair)]
    else:
        sig.operands.append((gu, pair))
    t = _out_vals(node)[0]
    sig.outputs.append((tuple(int(s) for s in t.shape), pair if is_bwd else list(lead), t.dtype))
    sig.follow = 1 if is_bwd else 0
    return sig


def _vocab_localize(arg_index: int, rows_arg: Optional[int] = None):
    def localize(node, ctx):
        args = list(node.args)
        while len(args) <= arg_index:
            args.append(0)
        args[arg_index] = ctx.shard_offset("vocab")
        if rows_arg is not None:
            args[rows_arg] = ctx.local_size("vocab")
        return tuple(args), dict(node.kwargs)
    return localize


def rule_ab_dropout(node: fx.Node) -> OpSig:
    """dropout(x, p, seed, stream, global_shape, offsets): pointwise in x; every dim may be sharded because the kernel
    keys the mask by the GLOBAL element index -- the localisation hook adds this shard's first coordinate per dim."""
    x, seed = node.args[0], node.args[2]
    sig = OpSig()
    o = _out_vals(node)[0]
    shape = tuple(int(s) for s in o.shape)
    labels = [sig.new(s) for s in shape]
    sig.operands.append((x, list(labels)))
    if isinstance(seed, fx.Node):
        sig.operands.append((seed, [sig.new(s, NOSHARD) for s in _shape(seed)]))
    sig.outputs.append((shape, list(labels), o.dtype))
    sig.named = {f"d{i}": l for i, l in enumerate(labels)}
    sig.follow = 0
    sig.zero_compatible = False

    def localize(node, ctx):
        args = list(node.args)
        base = list(args[5])
        args[5] = [int(b) + int(ctx.shard_offset(f"d{i}")) for i, b in enumerate(base)]
        return tuple(args), dict(node.kwargs)

    sig.localize = localize
    return sig


def rule_sdpa(node: fx.Node) -> OpSig:
    """torch's fused scaled-dot-product-attention ops (forward and backward, CPU / flash / efficient / cuDNN variants
    reached through nn.MultiheadAttention, F.scaled_dot_product_attention, ...): independent per (batch, head), so
    those two leading dims of every [B, H, ...] operand and result are shardable; sequence and head_dim are not.
    Small bookkeeping tensors (philox state, cumulative lengths) are replicated."""
    q = next(a for a in _tensor_args(node) if len(_shape(a)) == 4 and a is not node.args[0]) if \
        "backward" in str(node.target) else node.args[0]
    B, H = _shape(q)[0], _shape(q)[1]
    sig = OpSig()
    lb, lh = sig.new(B), sig.new(H)

    def labels_of(shape):
        out = []
        for d, sz in enumerate(shape):
            if d == 0 and len(shape) >= 3 and sz == B and B > 1:
                out.append(lb)
            elif d == 1 and len(shape) >= 3 and sz == H and shape[0] in (B, 1) and H > 1:
                out.append(lh)
            else:
                out.append(sig.new(sz, NOSHARD) if sz > 1 else -1)
        return out
    for a in _tensor_args(node):
        sig.operands.append((a, labels_of(_shape(a))))
    for o in _out_vals(node):
        shp = tuple(int(x) for x in o.shape)
        sig.outputs.append((shp, labels_of(shp), o.dtype))
    sig.follow = -1        # a heavy leader: must be spread over the whole mesh (batch and / or heads), never replicated
    S_, D = _shape(q)[2], _shape(q)[3]
    sig.flops = 4.0 * B * H * S_ * S_ * D
    return sig


def rule_ab_embedding(node: fx.Node) -> OpSig:
    ids, wte = node.args[0], node.args[1]
    sig = OpSig()
    idl = [sig.new(s) for s in _shape(ids)]
    lv, lh = sig.new(_shape(wte)[0]), sig.new(_shape(wte)[1])
    sig.operands += [(ids, idl), (wte, [lv, lh])]
    o = _out_vals(node)[0]
    sig.outputs.append((tuple(int(s) for s in o.shape), idl + [lh], o.dtype))
    sig.named = {"vocab": lv}
    sig.localize = _vocab_localize(2)
    sig.flops = 1.0  # leader: the vocab-parallel vs replicated choice is a real decision
    return sig


def rule_ab_embedding_bwd(node: fx.Node) -> OpSig:
    ids, dy = node.args[0], node.args[1]
    sig = OpSig()
    idl = [sig.new(s) for s in _shape(ids)]
    lh = sig.new(_shape(dy)[-1])
    o = _out_vals(node)[0]
    lv = sig.new(o.shape[0])
    sig.operands += [(ids, idl), (dy, idl + [lh])]
    sig.outputs.append((tuple(int(s) for s in o.shape), [lv, lh], o.dtype))
    sig.named = {"vocab": lv}
    sig.localize = _vocab_localize(3, rows_arg=2)
    sig.flops = 1.0
    return sig


def rule_ab_cross_entropy(node: fx.Node) -> OpSig:
    logits, labels = node.args[0], node.args[1]
    sig = OpSig()
    ls = _shape(logits)
    lead = _lead_labels(sig, ls[:-1])
    lv = sig.new(ls[-1], NOSHARD)
    sig.operands += [(logits, lead + [lv]), (labels, list(lead))]
    vals = _val(node)
    sig.outputs.append((tuple(int(s) for s in vals[0].shape), list(lead), vals[0].dtype))
    # stats [T,3]: T is the flattened token dim -> shardable only when logits are 2-D
    tl = [lead[0]] if len(lead) == 1 else [sig.new(vals[1].shape[0], NOSHARD)]
    sig.outputs.append((tuple(int(s) for s in vals[1].shape), tl + [sig.new(3, NOSHARD)], vals[1].dtype))
    sig.follow = 0
    return sig


def rule_ab_cross_entropy_bwd(node: fx.Node) -> OpSig:
    logits, labels, stats, dloss = node.args[:4]
    sig = OpSig()
    ls = _shape(logits)
    lead = _lead_labels(sig, ls[:-1])
    lv = sig.new(ls[-1], NOSHARD)
    tl = [lead[0]] if len(lead) == 1 else [sig.new(_shape(stats)[0], NOSHARD)]
    sig.operands += [(logits, lead + [lv]), (labels, list(lead)), (stats, tl + [sig.new(3, NOSHARD)]),
                     (dloss, list(lead))]
    o = _out_vals(node)[0]
    sig.outputs.append((tuple(int(s) for s in o.shape), lead + [lv], o.dtype))
    sig.follow = 0
    return sig


def rule_ab_bmm(node: fx.Node) -> OpSig:
    a, b, ta, tb = node.args[:4]
    sig = OpSig()
    ash, bsh = _shape(a), _shape(b)
    lb = sig.new(ash[0])
    M, K = (ash[2], ash[1]) if ta else (ash[1], ash[2])
    N = bsh[2] if tb else bsh[1]
    lm, lk, ln = sig.new(M), sig.new(K), sig.new(N)
    sig.operands += [(a, [lb, lk, lm] if ta else [lb, lm, lk]), (b, [lb, lk, ln] if tb else [lb, ln, lk])]
    o = _out_vals(node)[0]
    sig.outputs.append((tuple(int(s) for s in o.shape), [lb, lm, ln], o.dtype))
    sig.flops = 2.0 * ash[0] * M * K * N
    return sig


def _moe_route_labels(sig: OpSig, expert: fx.Node):
    G, S, K = _shape(expert)
    lg, ls, lk = sig.new(G), sig.new(S, NOSHARD), sig.new(K, NOSHARD)
    return lg, ls, lk


def rule_ab_moe_route(node: fx.Node) -> OpSig:
    gates = node.args[0]
    sig = OpSig()
    G, S, E = _shape(gates)
    lg, ls, le, lk = sig.new(G), sig.new(S, NOSHARD), sig.new(E, NOSHARD), sig.new(2, NOSHARD)
    sig.operands.append((gates, [lg, ls, le]))
    for o in _out_vals(node):
        sig.outputs.append((tuple(int(s) for s in o.shape), [lg, ls, lk], o.dtype))
    sig.follow = 0
    return sig


def rule_ab_moe_dispatch(node: fx.Node) -> OpSig:
    """x [G,S,M] -> d [E, G*C, M].  Groups route independently, so G (the major part of the G*C dim)
    and M are shardable; expert parallelism is the all-to-all resharding of d from G- to E-sharded."""
    x, expert, slot, weight = node.args[:4]
    sig = OpSig()
    lg, ls, lk = _moe_route_labels(sig, expert)
    lm = sig.new(_shape(x)[2])
    le = sig.new(node.args[4], NOSHARD)
    sig.operands += [(x, [lg, ls, lm]), (expert, [lg, ls, lk]), (slot, [lg, ls, lk])]
    if _is_tensor_node(weight):
        sig.operands.append((weight, [lg, ls, lk]))
    o = _out_vals(node)[0]
    sig.outputs.append((tuple(int(s) for s in o.shape), [le, lg, lm], o.dtype))
    sig.follow = 0
    return sig


def rule_ab_moe_combine(node: fx.Node) -> OpSig:
    eo, expert, slot, weight = node.args[:4]
    sig = OpSig()
    lg, ls, lk = _moe_route_labels(sig, expert)
    es = _shape(eo)
    le, lm = sig.new(es[0], NOSHARD), sig.new(es[2])
    sig.operands += [(eo, [le, lg, lm]), (expert, [lg, ls, lk]), (slot, [lg, ls, lk])]
    if _is_tensor_node(weight):
        sig.operands.append((weight, [lg, ls, lk]))
    o = _out_vals(node)[0]
    sig.outputs.append((tuple(int(s) for s in o.shape), [lg, ls, lm], o.dtype))
    # leader: the expert outputs arrive expert-sharded, tokens leave group-sharded -- following `eo` would tie the
    # combine to the expert GEMM's strategy and force an all-gather instead of the all-to-all
    sig.follow = -1
    sig.flops = 1.0
    return sig


def rule_ab_moe_combine_wgrad(node: fx.Node) -> OpSig:
    dout, eo, expert, slot = node.args[:4]
    sig = OpSig()
    lg, ls, lk = _moe_route_labels(sig, expert)
    es = _shape(eo)
    le, lm = sig.new(es[0], NOSHARD), sig.new(es[2])   # M is contracted: sharding it = partial sums
    sig.operands += [(dout, [lg, ls, lm]), (eo, [le, lg, lm]), (expert, [lg, ls, lk]), (slot, [lg, ls, lk])]
    o = _out_vals(node)[0]
    sig.outputs.append((tuple(int(s) for s in o.shape), [lg, ls, lk], o.dtype))
    sig.follow = 0
    return sig


def rule_ab_marker(node: fx.Node) -> OpSig:
    xs = node.args[0]
    sig = OpSig()
    vals = _val(node)
    for x, o in zip(xs, vals):
        labels = [sig.new(s) for s in _shape(x)]
        sig.operands.append((x, labels))
        sig.outputs.append((tuple(int(s) for s in o.shape), list(labels), o.dtype))
    sig.follow = 0 if xs else -1
    sig.per_operand_follow = True  # output i follows operand i (handled by the graph builder)
    return sig


def rule_ab_fused_adamw(node: fx.Node) -> OpSig:
    # expanded by the graph builder into one element-wise group per parameter
    raise RuntimeError("fused_adamw_ is expanded by the graph builder")


# ------------------------------------------------------------------------------------------------
# registry
# ------------------------------------------------------------------------------------------------
RULES: Dict[Any, Callable[[fx.Node], OpSig]] = {}


def _reg(targets, rule):
    for t in targets:
        RULES[t] = rule


_reg([aten.t.default, aten.transpose.int, aten.permute.default], rule_permute)
_reg([aten.view.default, aten._unsafe_view.default, aten.reshape.default, aten.squeeze.dim, aten.squeeze.dims,
      aten.squeeze.default, aten.unsqueeze.default, aten.flatten.using_ints, aten.unflatten.int], rule_reshape)
_reg([aten.expand.default], rule_expand)
_reg([aten.sum.dim_IntList, aten.sum.default], lambda n: rule_reduce(n, "sum"))
_reg([aten.amax.default, aten.max.default], lambda n: rule_reduce(n, "max"))
_reg([aten.amin.default, aten.min.default], lambda n: rule_reduce(n, "min"))
_reg([aten.mm.default, aten.bmm.default, aten.addmm.default], rule_mm)
_reg([aten._softmax.default, aten._log_softmax.default], rule_softmax)
_reg([aten._softmax_backward_data.default, aten._log_softmax_backward_data.default],
     lambda n: _dimwise(n, n.args[0], [n.args[2]], extra_operands=[(n.args[1], {d: d for d in range(len(_shape(n.args[1])))})]))
_reg([aten.native_layer_norm.default], rule_native_layer_norm)
_reg([aten.embedding.default], rule_embedding)
_reg([aten.embedding_dense_backward.default], rule_embedding_dense_backward)
_reg([aten.gather.default], rule_dim_op(1, extra=(2,)))
_reg([aten.scatter.src, aten.scatter.value, aten.scatter_add.default], rule_dim_op(1, extra=(2, 3)))
_reg([aten.index_select.default], rule_dim_op(1))
_reg([aten.cumsum.default, aten.cumprod.default, aten.argmax.default, aten.argmin.default, aten.flip.default],
     rule_dim_op(1, default_dim=None))
_reg([aten.sort.default], rule_dim_op(1, default_dim=-1))
_reg([aten.topk.default], rule_dim_op(2, default_dim=-1))          # topk(x, k, dim=-1, ...)
_reg([aten.roll.default], rule_dim_op(2, default_dim=None))        # roll(x, shifts, dims=[])
_reg([aten.slice.Tensor, aten.slice_backward.default, aten.select_backward.default, aten.split_with_sizes.default,
      aten.split.Tensor, aten.unbind.int, aten.chunk.default, aten.narrow.default], None)  # filled below
_reg([aten.select.int], rule_select)
_reg([aten.cat.default], rule_cat)
_reg([aten.full.default, aten.zeros.default, aten.ones.default, aten.empty.memory_format, aten.arange.default,
      aten.arange.start, aten.arange.start_step, aten.scalar_tensor.default, aten.rand.default, aten.randn.default],
     rule_constant)
_reg([operator.getitem], rule_getitem)
_reg([aten.convolution.default], rule_convolution)
_reg([aten.convolution_backward.default], rule_convolution_backward)
_reg([aten.max_pool2d_with_indices.default, aten.avg_pool2d.default, aten._adaptive_avg_pool2d.default,
      aten.max_pool2d_with_indices_backward.default, aten.avg_pool2d_backward.default,
      aten._adaptive_avg_pool2d_backward.default, aten.upsample_nearest2d.default,
      aten.upsample_nearest2d_backward.default], rule_pool)
_reg([aten.native_batch_norm.default, aten._native_batch_norm_legit.default,
      aten._native_batch_norm_legit_no_training.default, aten._native_batch_norm_legit_functional.default],
     rule_batch_norm)
_reg([aten.native_group_norm.default], rule_group_norm)
_reg([aten.constant_pad_nd.default], rule_constant_pad)


def _slice_rule(node: fx.Node) -> OpSig:
    t = node.target
    if t in (aten.slice.Tensor, aten.narrow.default):
        dim = node.args[1] if len(node.args) > 1 else 0
        return _dimwise(node, node.args[0], [dim])
    if t in (aten.split_with_sizes.default, aten.split.Tensor, aten.chunk.default):
        dim = node.args[2] if len(node.args) > 2 else 0
        return _dimwise(node, node.args[0], [dim])
    if t == aten.unbind.int:
        return rule_replicated(node)
    if t == aten.slice_backward.default:
        dim = node.args[2]
        sig = _dimwise(node, node.args[0], [dim])

        def localize(node, ctx):
            args = list(node.args)
            args[1] = list(ctx.local_out_shape(0))
            return tuple(args), dict(node.kwargs)
        sig.localize = localize
        return sig
    if t == aten.select_backward.default:
        # grad [..] -> zeros(input_sizes) with grad written at index along `dim`: out dim d <- grad dim d (d < dim)
        # or d - 1 (d > dim); `dim` itself is a new unsharded dim
        sizes, dim = node.args[1], node.args[2]
        nd = len(sizes)
        dim %= nd
        out_map = {d: (d if d < dim else d - 1) for d in range(nd) if d != dim}
        sig = _dimwise(node, node.args[0], [], out_map=out_map)

        def localize_sel(node, ctx):
            args = list(node.args)
            args[1] = list(ctx.local_out_shape(0))
            return tuple(args), dict(node.kwargs)
        sig.localize = localize_sel
        return sig
    return rule_replicated(node)


for _t in (aten.slice.Tensor, aten.slice_backward.default, aten.select_backward.default,
           aten.split_with_sizes.default, aten.split.Tensor, aten.unbind.int, aten.chunk.default,
           aten.narrow.default):
    RULES[_t] = _slice_rule

import alpa_b200.ops  # noqa: E402,F401  (registers the alpa_b200:: primitives)
_ab = torch.ops.alpa_b200
_reg([_ab.linear.default, _ab.linear_act.default], rule_ab_linear)
_reg([_ab.linear_dgrad.default, _ab.linear_dgrad_act.default, _ab.linear_dgrad_add.default], rule_ab_linear_dgrad)
_reg([_ab.linear_wgrad.default], rule_ab_linear_wgrad)
_reg([_ab.bias_grad.default], rule_ab_bias_grad)
_reg([_ab.act_bwd.default], rule_pointwise)
_reg([_ab.dropout.default], rule_ab_dropout)
_SDPA_OPS = [getattr(aten, n).default for n in (
    "_scaled_dot_product_flash_attention_for_cpu", "_scaled_dot_product_flash_attention_for_cpu_backward",
    "_scaled_dot_product_efficient_attention", "_scaled_dot_product_efficient_attention_backward",
    "_scaled_dot_product_flash_attention", "_scaled_dot_product_flash_attention_backward",
    "_scaled_dot_product_cudnn_attention", "_scaled_dot_product_cudnn_attention_backward") if hasattr(aten, n)]
_reg(_SDPA_OPS, rule_sdpa)
_reg([_ab.layer_norm.default, _ab.add_layer_norm.default, _ab.rms_norm.default, _ab.add_rms_norm.default],
     rule_ab_layer_norm)
_reg([_ab.layer_norm_bwd.default, _ab.rms_norm_bwd.default], rule_ab_layer_norm_bwd)
_reg([_ab.rotary_packed.default], rule_ab_rotary_packed)
_reg([_ab.swiglu.default, _ab.swiglu_bwd.default], rule_ab_swiglu)
_reg([_ab.attention.default], rule_ab_attention)
_reg([_ab.attention_bwd.default], rule_ab_attention_bwd)
_reg([_ab.attention_cached.default], rule_ab_attention_cached)
_reg([_ab.attention_gqa_packed.default, _ab.attention_gqa_packed_bwd.default], rule_ab_attention_gqa_packed)
_reg([_ab.embedding.default], rule_ab_embedding)
_reg([_ab.embedding_bwd.default], rule_ab_embedding_bwd)
_reg([_ab.cross_entropy.default], rule_ab_cross_entropy)
_reg([_ab.cross_entropy_bwd.default], rule_ab_cross_entropy_bwd)
_reg([_ab.pipeline_marker.default], rule_ab_marker)
_reg([_ab.bmm.default], rule_ab_bmm)
_reg([_ab.moe_top2_route.default], rule_ab_moe_route)
_reg([_ab.moe_dispatch.default], rule_ab_moe_dispatch)
_reg([_ab.moe_combine.default], rule_ab_moe_combine)
_reg([_ab.moe_combine_wgrad.default], rule_ab_moe_combine_wgrad)

_IDENTITY_LIKE = {aten.detach.default, aten.alias.default, aten.clone.default, aten._to_copy.default,
                  aten.lift_fresh_copy.default, aten.contiguous.default, aten.ones_like.default,
                  aten.zeros_like.default, aten.full_like.default, aten.empty_like.default,
                  aten.rand_like.default, aten.randn_like.default, aten.native_dropout.default,
                  aten.bernoulli.p, aten.copy.default, aten.new_zeros.default, aten.new_ones.default}


def _pad_none_outputs(node: fx.Node, sig: OpSig) -> OpSig:
    """Tuple-valued ops may return None for masked-out results (convolution_backward's output_mask): keep the
    tuple positions by inserting scalar dummies so `getitem` indices address the right output."""
    v = _val(node)
    if isinstance(v, (list, tuple)) and any(not isinstance(t, torch.Tensor) for t in v):
        n_tensor = sum(isinstance(t, torch.Tensor) for t in v)
        if len(sig.outputs) == n_tensor:
            it = iter(sig.outputs)
            sig.outputs = [next(it) if isinstance(t, torch.Tensor) else ((), [], torch.float32) for t in v]
            if sig.output_depends is not None and len(sig.output_depends) == n_tensor:
                dit = iter(sig.output_depends)
                sig.output_depends = [next(dit) if isinstance(t, torch.Tensor) else [] for t in v]
    return sig


def signature_of(node: fx.Node) -> OpSig:
    """The sharding signature of a call_function node."""
    t = node.target
    rule = RULES.get(t)
    if rule is not None:
        return _pad_none_outputs(node, rule(node))
    if t in _IDENTITY_LIKE:
        return rule_pointwise(node)
    tags = getattr(t, "tags", None)
    if tags is not None and torch.Tag.pointwise in tags:
        return rule_pointwise(node)
    return rule_replicated(node)


def is_known(node: fx.Node) -> bool:
    t = node.target
    tags = getattr(t, "tags", None)
    return t in RULES or t in _IDENTITY_LIKE or (tags is not None and torch.Tag.pointwise in tags)
