"""FLOP / "heavy op" statistics of traced graphs (reference: alpa/pipeline_parallel/layer_stats.py:
eqn_flops:12, heavy_count:49, is_nontrivial:59, log_layer_slicing_stats:91)."""
from __future__ import annotations

import logging
from typing import Dict, List, Sequence

import torch
from torch import fx

from alpa_b200.parallel.shard import signatures as S

logger = logging.getLogger(__name__)

_HEAVY = None


def _heavy_targets():
    global _HEAVY
    if _HEAVY is None:
        a, ab = torch.ops.aten, torch.ops.alpa_b200
        _HEAVY = {a.mm.default, a.bmm.default, a.addmm.default, a.convolution.default, a.convolution_backward.default,
                  ab.linear.default, ab.linear_act.default, ab.linear_dgrad.default, ab.linear_dgrad_act.default, ab.linear_dgrad_add.default,
                  ab.linear_wgrad.default, ab.attention.default, ab.attention_bwd.default,
                  ab.attention_qkvpacked.default, ab.attention_qkvpacked_bwd.default,
                  ab.attention_gqa_packed.default, ab.attention_gqa_packed_bwd.default, ab.bmm.default}
    return _HEAVY


def node_flops(node: fx.Node) -> float:
    """FLOPs of one graph node from its sharding signature (2*M*N*K for GEMM-shaped ops, 0 for glue)."""
    if node.op != "call_function":
        return 0.0
    try:
        return max(0.0, float(S.signature_of(node).flops))
    except Exception:  # noqa: BLE001
        return 0.0


def heavy_count(node: fx.Node) -> int:
    """1 for matmul/conv/attention nodes (the ops layer clustering balances), else 0."""
    return int(node.op == "call_function" and node.target in _heavy_targets())


def is_nontrivial(node: fx.Node) -> bool:
    return heavy_count(node) > 0


def graph_stats(nodes: Sequence[fx.Node]) -> Dict[str, float]:
    return {"flops": sum(node_flops(n) for n in nodes), "heavy": sum(heavy_count(n) for n in nodes),
            "ops": sum(1 for n in nodes if n.op == "call_function")}


def log_layer_slicing_stats(layers: Sequence[Sequence[fx.Node]]) -> List[Dict[str, float]]:
    stats = [graph_stats(l) for l in layers]
    total = sum(s["flops"] for s in stats) or 1.0
    for i, s in enumerate(stats):
        logger.info("layer %d: %.3f GFLOP (%.1f%%), %d heavy ops, %d ops", i, s["flops"] / 1e9,
                    100 * s["flops"] / total, s["heavy"], s["ops"])
    return stats
