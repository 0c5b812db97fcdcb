"""Clusters, device meshes, communicators and distributed arrays.

Reference: alpa/device_mesh.py (DeviceCluster:2131, VirtualPhysicalMesh:1792, PhysicalDeviceMesh:633,
LocalPhysicalDeviceMesh:860, DistributedPhysicalDeviceMesh:979, DistributedArray:1509,
ReplicatedDistributedArray:1697, PhysicalDeviceMeshGroup:1979, globals :2308-2406).

H100-native process model: **one process per GPU, SPMD** (torchrun / mp.spawn), no Ray driver and no
remote buffer table -- every rank runs the same Python program, owns the shards of its own GPU and
executes the same statically planned program.  Two execution backends share one executor:

* ``DistCommunicator``     -- real multi-process meshes over ``torch.distributed`` (nccl on GPUs,
                              gloo on CPU); each process has exactly one local device.
* ``EmulatedCommunicator`` -- all logical devices live in this process (a list of shards per array);
                              used by ``cluster="local"`` with ``num_devices>1`` and by device-free
                              tests, the analogue of the reference slicing one host into several meshes.
"""
from __future__ import annotations

import itertools
import os
import threading
from typing import Any, Dict, List, Optional, Sequence, Tuple

import weakref
import numpy as np
import torch
import torch.distributed as dist

from alpa_b200.global_env import global_config
from alpa_b200.sharding import LogicalDeviceMesh, ShardingSpec

########################################
# communicators
########################################


def _groups_along(logical_mesh: LogicalDeviceMesh, axes: Sequence[int]) -> List[Tuple[int, ...]]:
    """Partition the mesh's device ids into groups that vary only along `axes` (row-major order)."""
    shape = logical_mesh.shape
    other = [a for a in range(len(shape)) if a not in axes]
    groups = []
    for oc in itertools.product(*[range(shape[a]) for a in other]):
        g = []
        for ac in itertools.product(*[range(shape[a]) for a in axes]):
            c = [0] * len(shape)
            for a, v in zip(other, oc):
                c[a] = v
            for a, v in zip(axes, ac):
                c[a] = v
            g.append(int(logical_mesh.id_mesh[tuple(c)]))
        groups.append(tuple(g))
    return groups


class GradBucket:
    """Run-time state of one static gradient bucket of a lowered program (parallel/shard/lowering.py:
    `_plan_grad_buckets`): a persistent flat buffer per local device, one view per member gradient, and
    `reduce_async()` = ONE in-place sum all-reduce of the whole buffer.  Addresses never change, so a CUDA graph of
    the step replays it.  (reference: XLA's all-reduce combiner + NCCL thunk, gpu_compiler.cc:663-679.)"""

    kind = "all-reduce"

    def __init__(self, comm, plan, logical_mesh, devices, flats: Optional[List[torch.Tensor]] = None):
        self.comm, self.plan, self.mesh = comm, plan, logical_mesh
        self.flat = flats if flats is not None else [torch.zeros(plan.numel, dtype=plan.dtype, device=d) for d in devices]
        self.views = [[f[off:off + n].view(shape) for f in self.flat] for (_, off, n, shape, _sub) in plan.members]

    def reduce_async(self):
        asyn = getattr(self.comm, "all_reduce_async_inplace", None)
        if asyn is not None:
            return asyn(self.flat, self.mesh, list(self.plan.axes))
        outs = self.comm.all_reduce(self.flat, self.mesh, list(self.plan.axes), "sum")
        for f, o in zip(self.flat, outs):
            if o.data_ptr() != f.data_ptr():
                f.copy_(o)
        return None


class EmulatedCommunicator:
    """Collectives over a list holding *every* device's tensor (position = device order of the mesh)."""

    def __init__(self, device_ids: Sequence[int]):
        self.device_ids = list(device_ids)
        self.pos = {d: i for i, d in enumerate(self.device_ids)}
        self.stats: Dict[str, int] = {}

    def _count(self, name):
        self.stats[name] = self.stats.get(name, 0) + 1

    def all_reduce(self, xs, logical_mesh, axes, op="sum"):
        self._count("all-reduce")
        out = list(xs)
        for g in _groups_along(logical_mesh, axes):
            idx = [self.pos[d] for d in g]
            stacked = torch.stack([xs[i] for i in idx])
            if op == "sum":
                r = stacked.sum(0)
            elif op == "max":
                r = stacked.max(0).values
            elif op == "min":
                r = stacked.min(0).values
            else:
                raise ValueError(op)
            for i in idx:
                out[i] = r.clone()
        return out

    def all_gather(self, xs, logical_mesh, axis, dim):
        self._count("all-gather")
        out = list(xs)
        for g in _groups_along(logical_mesh, [axis]):
            idx = [self.pos[d] for d in g]
            r = torch.cat([xs[i] for i in idx], dim=dim)
            for i in idx:
                out[i] = r.clone()
        return out

    def reduce_scatter(self, xs, logical_mesh, axis, dim):
        self._count("reduce-scatter")
        out = list(xs)
        for g in _groups_along(logical_mesh, [axis]):
            idx = [self.pos[d] for d in g]
            r = torch.stack([xs[i] for i in idx]).sum(0)
            chunks = torch.chunk(r, len(idx), dim=dim)
            for k, i in enumerate(idx):
                out[i] = chunks[k].contiguous()
        return out

    def all_to_all(self, xs, logical_mesh, axis, split_dim, concat_dim):
        self._count("all-to-all")
        out = list(xs)
        for g in _groups_along(logical_mesh, [axis]):
            idx = [self.pos[d] for d in g]
            pieces = [torch.chunk(xs[i], len(idx), dim=split_dim) for i in idx]
            for k, i in enumerate(idx):
                out[i] = torch.cat([pieces[j][k] for j in range(len(idx))], dim=concat_dim).contiguous()
        return out

    # asynchronous variants: the emulated mesh runs them eagerly (no handle), which keeps the lowered program --
    # asynchronous gradient sync, hoisted parameter all-gathers, static gradient buckets -- identical to the GPU one
    def all_reduce_async(self, xs, logical_mesh, axes, op="sum"):
        return self.all_reduce(xs, logical_mesh, axes, op), None

    def all_gather_async(self, xs, logical_mesh, axis, dim):
        return self.all_gather(xs, logical_mesh, axis, dim), None

    def reduce_scatter_async(self, xs, logical_mesh, axis, dim):
        return self.reduce_scatter(xs, logical_mesh, axis, dim), None

    def barrier(self):
        pass


class DistCommunicator:
    """Collectives over torch.distributed; every process holds exactly one shard (lists of length 1)."""

    _group_cache: Dict[Tuple[int, ...], Any] = {}
    _lock = threading.Lock()

    def __init__(self, device_ids: Sequence[int]):
        self.device_ids = list(device_ids)
        self.rank = dist.get_rank()
        self.stats: Dict[str, int] = {}

    def _count(self, name):
        self.stats[name] = self.stats.get(name, 0) + 1

    @classmethod
    def get_group(cls, ranks: Tuple[int, ...]):
        """Process group for `ranks`.  NOTE: creation is collective over the world; every rank reaches
        this call with the same arguments in the same order because planning is deterministic."""
        ranks = tuple(ranks)
        if len(ranks) == dist.get_world_size() and ranks == tuple(range(len(ranks))):
            return dist.group.WORLD
        with cls._lock:
            if ranks not in cls._group_cache:
                cls._group_cache[ranks] = dist.new_group(list(ranks))
            return cls._group_cache[ranks]

    def ensure_groups(self, logical_mesh: LogicalDeviceMesh):
        """Eagerly create the groups of every mesh axis (and both) -- on *all* world ranks."""
        nd = len(logical_mesh.shape)
        for axes in [[a] for a in range(nd)] + ([list(range(nd))] if nd > 1 else []):
            for g in _groups_along(logical_mesh, axes):
                if len(g) > 1:
                    self.get_group(g)

    def _my_group(self, logical_mesh, axes):
        for g in _groups_along(logical_mesh, axes):
            if self.rank in g:
                if len(g) > 1:
                    # create sibling groups too, in a fixed order, to keep new_group collective-safe
                    for gg in _groups_along(logical_mesh, axes):
                        self.get_group(gg)
                return g
        raise RuntimeError(f"rank {self.rank} not in mesh {logical_mesh.flatten_ids}")

    def all_reduce(self, xs, logical_mesh, axes, op="sum"):
        self._count("all-reduce")
        g = self._my_group(logical_mesh, axes)
        if len(g) == 1:
            return xs
        x = xs[0].contiguous()
        rop = {"sum": dist.ReduceOp.SUM, "max": dist.ReduceOp.MAX, "min": dist.ReduceOp.MIN}[op]
        dist.all_reduce(x, op=rop, group=self.get_group(g))
        return [x]

    def all_reduce_async(self, xs, logical_mesh, axes, op="sum"):
        """Launch the all-reduce on NCCL's own stream and return (tensors, work); the caller waits on
        `work` right before the first consumer, so the reduction overlaps the remaining backward pass
        (K10 of SURVEY.md §2.5: the reference serialises gradient sync after backward)."""
        self._count("all-reduce")
        g = self._my_group(logical_mesh, axes)
        if len(g) == 1:
            return xs, None
        x = xs[0].contiguous()
        if op == "sum" and x.is_cuda and x.dtype == torch.bfloat16:
            red = self._nvls_reducer(g)
            if red is not None:
                h = red.add(x)
                if h is not None:
                    return [x], h
        rop = {"sum": dist.ReduceOp.SUM, "max": dist.ReduceOp.MAX, "min": dist.ReduceOp.MIN}[op]
        work = dist.all_reduce(x, op=rop, group=self.get_group(g), async_op=True)
        return [x], work

    def all_reduce_async_inplace(self, xs, logical_mesh, axes):
        """In-place sum all-reduce of a persistent buffer on NCCL's stream; returns the work handle (or None)."""
        self._count("all-reduce")
        g = self._my_group(logical_mesh, axes)
        if len(g) == 1:
            return None
        return dist.all_reduce(xs[0], op=dist.ReduceOp.SUM, group=self.get_group(g), async_op=True)

    def make_grad_bucket(self, plan, logical_mesh, ndev, device, all_plans=None, program_key=None):
        """Bucket state for this process: in-switch NVLS reduction of a symmetric-memory bucket (device-side
        barriers, graph-capturable) when enabled and available, otherwise a plain buffer + one NCCL all-reduce."""
        from alpa_b200.global_env import global_config
        g = self._my_group(logical_mesh, list(plan.axes))
        if (getattr(global_config, "use_nvls_grad_allreduce", False) and device.type == "cuda" and
                plan.dtype == torch.bfloat16 and 1 < len(g) <= 8):
            try:
                from alpa_b200 import ops
                from alpa_b200.collective.fused import NvlsBucketArena
                if ops.native_available():
                    arenas = self.__dict__.setdefault("_nvls_arenas", {})
                    key = (program_key, tuple(g))
                    if key not in arenas:
                        plans = [p for p in (all_plans or [plan]) if p.dtype == torch.bfloat16 and
                                 tuple(p.axes) == tuple(plan.axes)]
                        arenas[key] = NvlsBucketArena(self.get_group(g), plans)
                    return arenas[key].bucket(self, plan, logical_mesh)
            except Exception as e:  # noqa: BLE001
                if not self.__dict__.get("_nvls_bucket_warned"):
                    self.__dict__["_nvls_bucket_warned"] = True
                    import logging
                    logging.getLogger(__name__).warning("NVLS gradient buckets unavailable (%s); using NCCL", e)
        return GradBucket(self, plan, logical_mesh, [device] * ndev)

    def _nvls_reducer(self, g):
        """Bucketed in-switch (NVLS) gradient all-reduce for this device group, or None (-> NCCL)."""
        from alpa_b200.global_env import global_config
        nvls = getattr(global_config, "use_nvls_grad_allreduce", False)
        bucketed = getattr(global_config, "use_bucketed_grad_allreduce", False)
        if not (nvls or bucketed):
            return None
        cache = self.__dict__.setdefault("_nvls", {})
        key = tuple(g)
        if key not in cache:
            try:
                from alpa_b200 import ops
                from alpa_b200.collective.fused import NvlsGradReducer
                if nvls and ops.native_available() and 1 < len(g) <= 8:
                    cache[key] = NvlsGradReducer(self.get_group(g), mode="nvls")
                else:
                    cache[key] = NvlsGradReducer(self.get_group(g), mode="nccl")
            except Exception as e:  # noqa: BLE001
                import logging
                logging.getLogger(__name__).warning("NVLS gradient all-reduce unavailable (%s); using NCCL", e)
                cache[key] = None
        return cache[key]

    def all_gather(self, xs, logical_mesh, axis, dim):
        self._count("all-gather")
        g = self._my_group(logical_mesh, [axis])
        if len(g) == 1:
            return xs
        x = xs[0].contiguous()
        n = len(g)
        if x.dim() == 0:
            x = x.reshape(1)
        out = torch.empty((n * x.shape[0],) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        dist.all_gather_into_tensor(out, x, group=self.get_group(g))
        if dim == 0:
            return [out]
        return [torch.cat(list(out.chunk(n, dim=0)), dim=dim)]

    def reduce_scatter(self, xs, logical_mesh, axis, dim):
        self._count("reduce-scatter")
        g = self._my_group(logical_mesh, [axis])
        if len(g) == 1:
            return xs
        n = len(g)
        x = xs[0]
        if dim != 0:
            x = torch.cat(torch.chunk(x, n, dim=dim), dim=0)
        x = x.contiguous()
        out = torch.empty((x.shape[0] // n,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        if x.device.type == "cpu":  # gloo has no reduce_scatter
            dist.all_reduce(x, group=self.get_group(g))
            out.copy_(torch.chunk(x, n, dim=0)[g.index(self.rank)])
        else:
            dist.reduce_scatter_tensor(out, x, group=self.get_group(g))
        return [out]

    def all_gather_async(self, xs, logical_mesh, axis, dim):
        """All-gather on NCCL's stream; returns (tensors, work).  Only dim-0 gathers run asynchronously (the
        concatenation of other dims needs the data)."""
        g = self._my_group(logical_mesh, [axis])
        x = xs[0]
        if len(g) == 1 or x.device.type == "cpu" or dim != 0 or x.dim() == 0:
            return self.all_gather(xs, logical_mesh, axis, dim), None
        self._count("all-gather")
        x = x.contiguous()
        out = torch.empty((len(g) * x.shape[0],) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        work = dist.all_gather_into_tensor(out, x, group=self.get_group(g), async_op=True)
        return [out], work

    def reduce_scatter_async(self, xs, logical_mesh, axis, dim):
        """Reduce-scatter on NCCL's stream; returns (shards, work) -- the caller waits right before the first use
        (ZeRO-2/3 gradient sync overlapped with the remaining backward pass)."""
        g = self._my_group(logical_mesh, [axis])
        x = xs[0]
        if len(g) == 1 or x.device.type == "cpu":
            return self.reduce_scatter(xs, logical_mesh, axis, dim), None
        self._count("reduce-scatter")
        n = len(g)
        if dim != 0:
            x = torch.cat(torch.chunk(x, n, dim=dim), dim=0)
        x = x.contiguous()
        out = torch.empty((x.shape[0] // n,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        work = dist.reduce_scatter_tensor(out, x, group=self.get_group(g), async_op=True)
        return [out], work

    def all_to_all(self, xs, logical_mesh, axis, split_dim, concat_dim):
        self._count("all-to-all")
        g = self._my_group(logical_mesh, [axis])
        if len(g) == 1:
            return xs
        n = len(g)
        ins = [c.contiguous() for c in torch.chunk(xs[0], n, dim=split_dim)]
        outs = [torch.empty_like(c) for c in ins]
        if xs[0].device.type == "cpu":
            # gloo: emulate with all_gather of the full list
            gathered = [torch.empty_like(xs[0].contiguous()) for _ in range(n)]
            dist.all_gather(gathered, xs[0].contiguous(), group=self.get_group(g))
            me = g.index(self.rank)
            outs = [torch.chunk(t, n, dim=split_dim)[me] for t in gathered]
        else:
            dist.all_to_all(outs, ins, group=self.get_group(g))
        return [torch.cat(outs, dim=concat_dim).contiguous()]

    # ---- fused compute + collective kernels over NVLink peer memory (alpa_b200/collective/fused.py)
    def fused_op(self, kind, site, args, logical_mesh, axis, target=None):
        """Run one fused (compute, collective) instruction of a lowered program, or return None when this
        communicator / these shapes are not served by a fused kernel (caller falls back to compute + NCCL)."""
        from alpa_b200.global_env import global_config
        if not global_config.use_fused_collectives or not torch.cuda.is_available():
            return None
        tensors = [a for a in args if isinstance(a, torch.Tensor)]
        if not tensors or not all(t.is_cuda for t in tensors):
            return None
        from alpa_b200 import ops
        if not ops.native_available():
            return None
        g = self._my_group(logical_mesh, [axis])
        n = len(g)
        if n == 1 or n > 8:
            return None
        bf16 = torch.bfloat16
        key = (site, kind)
        cache = self.__dict__.setdefault("_fused_sites", {})
        try:
            from alpa_b200.collective import fused as F
            group = self.get_group(g)
            if kind == "moe_dispatch_a2a":
                x, expert, slot, weight, E, C = args
                if x.dtype != bf16 or E % n or x.shape[2] % 8:
                    return None
                if key not in cache:
                    cache[key] = F.FusedMoEDispatch(group, E, x.shape[0], C, x.shape[2])
                return cache[key](x, expert, slot, weight)
            if kind in ("moe_combine_a2a", "moe_combine_wgrad_a2a"):
                eo = args[0] if kind == "moe_combine_a2a" else args[1]
                if eo.dtype != bf16 or eo.shape[2] % 8:
                    return None
                if key not in cache:
                    cache[key] = F.FusedMoECombine(group, eo.shape[0], eo.shape[1], eo.shape[2])
                if kind == "moe_combine_a2a":
                    return cache[key].combine(eo, args[1], args[2], args[3])
                return cache[key].combine_wgrad(args[0], eo, args[2], args[3])
            if kind == "linear_all_reduce":
                # y = all_reduce(x @ w^T [+ b on one rank]): the GEMM epilogue writes straight into a symmetric
                # buffer, the NVSwitch reduces it in place (multimem.ld_reduce / multimem.st); no NCCL, no staging copy
                ab = torch.ops.alpa_b200
                x, w = args[0], args[1]
                b = args[2] if (target == ab.linear.default and len(args) > 2) else None
                res = args[2] if (target == ab.linear_dgrad_add.default and len(args) > 2) else None
                if x.dtype != bf16:
                    return None
                trans_b = target in (ab.linear_dgrad.default, ab.linear_dgrad_add.default)   # dgrad: dy @ w (w is [N, K])
                x2 = x.reshape(-1, x.shape[-1])
                M = x2.shape[0]
                N = w.shape[1] if trans_b else w.shape[0]
                if (M * N) % (8 * n) or N % 8 or x2.shape[1] % 8 or not x2.is_contiguous() or not w.is_contiguous():
                    return None
                if key not in cache:
                    op = F.MultimemAllReduce(group, M * N)
                    if not op.available:
                        cache[key] = None
                    else:
                        cache[key] = op
                op = cache[key]
                if op is None:
                    return None
                out2 = op.tensor.view(M, N)
                if res is not None:          # accumulated gradient: added on the one device that received it
                    res = res.reshape(M, N)
                    if not res.is_contiguous():
                        return None
                ops.native_module().gemm(x2, w, False, trans_b, out=out2, bias=b, residual=res)
                op()                                                # barrier, in-switch reduce, barrier
                return out2.view(*x.shape[:-1], N)
            if kind == "all_gather_linear":
                # y = all_gather(x, rows) @ w^T (+ b, activation): rows pushed to every peer's symmetric buffer with
                # per-128-row flags, the GEMM's TMA producer waits for the block it is about to load.  The kernel pair
                # is validated stand-alone (profiles/r1_fused_collectives_*), this lowered call site has not run on
                # hardware yet: opt-in (`global_config.use_fused_allgather_linear`), otherwise all-gather + GEMM.
                if not getattr(global_config, "use_fused_allgather_linear", False):
                    return None
                ab = torch.ops.alpa_b200
                x, w = args[0], args[1]
                b = args[2] if len(args) > 2 else None
                act = args[3] if (target == ab.linear_act.default and len(args) > 3) else "none"
                if x.dtype != bf16:
                    return None
                x2 = x.reshape(-1, x.shape[-1])
                Ml, K = x2.shape
                if Ml % 128 or K % 8 or w.shape[0] % 8 or not x2.is_contiguous() or not w.is_contiguous():
                    return None
                if key not in cache:
                    cache[key] = F.FusedAllGatherLinear(group, Ml, K)
                lead = (x.shape[0] * n,) + tuple(x.shape[1:-1])
                if target == ab.linear_act.default:
                    z = torch.empty(n * Ml, w.shape[0], dtype=bf16, device=x.device)
                    y = cache[key](x2, w, b, act, aux_out=z)
                    return (y.view(*lead, w.shape[0]), z.view(*lead, w.shape[0]))
                return cache[key](x2, w, b).view(*lead, w.shape[0])
            if kind == "linear_reduce_scatter":
                # opt-in: at 8 GPUs the lowered ZeRO-2 step was SLOWER with the fused wgrad -> reduce-scatter kernels
                # (25.7 vs 21.9 ms, profiles/r1_fused_lowering_8gpu_v1.log), and every site owns a symmetric workspace
                # whose rendezvous costs seconds -- a pipeline stage with prefer_reduce_scatter has ~64 such sites
                if not getattr(global_config, "use_fused_linear_reduce_scatter", False):
                    return None
                ab = torch.ops.alpa_b200
                if target == ab.linear.default:
                    x, w = args[0], args[1]
                    b = args[2] if len(args) > 2 else None
                    if b is not None or x.dtype != bf16:
                        return None
                    x2 = x.reshape(-1, x.shape[-1])
                    M, N = x2.shape[0], w.shape[0]
                    lead = x.shape[:-1]
                    if lead[0] % n or M % (n * 32) or N % 8 or not x2.is_contiguous() or not w.is_contiguous():
                        return None
                    if key not in cache:
                        cache[key] = F.FusedLinearReduceScatter(group, M, N)
                    out = cache[key](x2, w)
                    return out.view(lead[0] // n, *lead[1:], N)
                if target == ab.linear_wgrad.default:
                    dy, x = args[0], args[1]
                    if dy.dtype != bf16:
                        return None
                    dy2, x2 = dy.reshape(-1, dy.shape[-1]), x.reshape(-1, x.shape[-1])
                    N, K = dy2.shape[1], x2.shape[1]          # dW [N, K] = dy^T x
                    if N % (n * 32) or K % 8 or N % 8 or not dy2.is_contiguous() or not x2.is_contiguous():
                        return None
                    if key not in cache:
                        cache[key] = F.FusedLinearReduceScatter(group, N, K)
                    return cache[key](dy2, x2, trans_a=True, trans_b=True)
        except RuntimeError as e:            # symmetric memory unavailable (no P2P / fabric): use NCCL
            if not self.__dict__.get("_fused_warned"):
                self.__dict__["_fused_warned"] = True
                import logging
                logging.getLogger(__name__).warning("fused collectives disabled: %s", e)
            return None
        return None

    def barrier(self):
        dist.barrier()


########################################
# physical meshes
########################################


class PhysicalDeviceMesh:
    """A set of devices (global ranks) that run one SPMD program.  shape = (num_hosts, devices/host)."""

    def __init__(self, devices: Sequence[int], num_hosts: int = 1, emulated: bool = False,
                 torch_device: Optional[torch.device] = None, parent=None):
        self.devices = list(devices)
        self.num_hosts = num_hosts
        assert len(self.devices) % num_hosts == 0
        self.num_devices_per_host = len(self.devices) // num_hosts
        self.emulated = emulated
        self.parent = parent
        if torch_device is None:
            torch_device = _default_torch_device()
        self.torch_device = torch_device
        if emulated:
            self.comm = EmulatedCommunicator(self.devices)
            self.local_devices = list(self.devices)
        else:
            self.comm = DistCommunicator(self.devices) if dist.is_initialized() else EmulatedCommunicator(self.devices)
            rank = dist.get_rank() if dist.is_initialized() else 0
            self.local_devices = [rank] if rank in self.devices else []
        self.launched = True

    # ---- shape ----
    @property
    def shape(self):
        return (self.num_hosts, self.num_devices_per_host)

    @property
    def num_devices(self):
        return len(self.devices)

    @property
    def device_ids(self):
        return self.devices

    @property
    def is_member(self) -> bool:
        return len(self.local_devices) > 0

    # ---- logical views ----
    def get_logical_mesh(self, mesh_shape: Optional[Sequence[int]] = None, mesh_alpha=None, mesh_beta=None,
                         mesh_topology=None, intra_host_bandwidth=None, inter_host_bandwidth=None):
        """Reference: PhysicalDeviceMesh.get_logical_mesh (device_mesh.py:686-770).  On a single
        NVSwitch domain both axes get equal beta; across hosts axis 0 is 10x slower by default."""
        if mesh_shape is None:
            mesh_shape = self.shape
        mesh_shape = tuple(int(x) for x in mesh_shape)
        assert int(np.prod(mesh_shape)) == self.num_devices, (mesh_shape, self.num_devices)
        id_mesh = np.array(self.devices).reshape(mesh_shape)
        if mesh_alpha is None:
            mesh_alpha = (1,) * len(mesh_shape)
        if mesh_beta is None:
            if self.num_hosts > 1 and len(mesh_shape) == 2 and mesh_shape[0] % self.num_hosts == 0:
                mesh_beta = (1, 0.1)
            else:
                mesh_beta = (1,) * len(mesh_shape)
        return LogicalDeviceMesh(self, id_mesh, mesh_alpha, mesh_beta)

    def get_default_logical_mesh(self):
        return self.get_logical_mesh((self.num_devices, 1) if self.num_hosts == 1 else self.shape)

    # ---- arrays ----
    def shard_tensor(self, x: torch.Tensor, logical_mesh: LogicalDeviceMesh, spec: ShardingSpec) -> "DistributedArray":
        """Slice a *global* tensor (identical on every rank) into this rank's shard(s)."""
        shards = []
        for d in self.local_devices:
            sl = spec.local_slices(x.shape, logical_mesh.coords_of(d))
            s = x[sl]
            if s.device != self.torch_device:
                # host -> device: asynchronous when the source is pinned (rows of a pinned batch)
                s = s.to(self.torch_device, non_blocking=True)
                shards.append(s if s.is_contiguous() else s.contiguous())
            else:
                shards.append(s.contiguous() if not s.is_contiguous() else s.clone())
        return DistributedArray(self, logical_mesh, tuple(x.shape), x.dtype, spec, shards)

    def sync_workers(self):
        if torch.cuda.is_available() and self.torch_device.type == "cuda":
            torch.cuda.synchronize()
        self.comm.barrier()

    def shutdown(self, forced=False):
        self.launched = False

    # memory statistics (reference: MeshHostWorker.get_memory_allocated etc., device_mesh.py:255-270)
    def get_memory_allocated(self):
        return torch.cuda.memory_allocated() if self.torch_device.type == "cuda" else 0

    def get_max_memory_allocated(self):
        return torch.cuda.max_memory_allocated() if self.torch_device.type == "cuda" else 0

    def get_available_memory(self):
        if self.torch_device.type == "cuda":
            free, _ = torch.cuda.mem_get_info()
            return free
        return 1 << 40

    def reset_memory_stats(self):
        if self.torch_device.type == "cuda":
            torch.cuda.reset_peak_memory_stats()

    def set_runtime_random_seed(self, seed: int):
        """(reference: PhysicalDeviceMesh.set_runtime_random_seed -- seeds the stateful RNG of the mesh workers)"""
        from alpa_b200.global_env import global_config
        global_config.runtime_random_seed = int(seed)
        torch.manual_seed(int(seed))
        if torch.cuda.is_available() and self.torch_device.type == "cuda":
            torch.cuda.manual_seed_all(int(seed))

    def get_remote_timer(self, timer_name: str):
        """(reference: get_remote_timer -- the worker-side timer of `timer_name`; one process per GPU here)"""
        from alpa_b200.timer import timers
        return timers(timer_name)

    def reset_remote_timer(self, timer_name: str):
        from alpa_b200.timer import timers
        timers(timer_name).reset()

    def get_remote_tracer(self):
        from alpa_b200.timer import tracer
        return tracer

    def sync_move_workers(self):
        """Wait for the background checkpoint movers (reference: DistributedPhysicalDeviceMesh.sync_move_workers)."""
        from alpa_b200 import serialization
        sync = getattr(serialization, "sync_move_workers", None) or getattr(serialization, "sync", None)
        if sync is not None:
            sync()

    def get_live_buffer_uuids(self) -> List[int]:
        """(reference: MeshHostWorker.get_live_buffer_uuids, used by tests/runtime/test_memory_leak.py)"""
        return get_live_buffer_uuids(self)

    def get_live_buffer_bytes(self) -> int:
        return get_live_buffer_bytes(self)

    def __repr__(self):
        return f"PhysicalDeviceMesh(devices={self.devices}, shape={self.shape}, emulated={self.emulated})"


LocalPhysicalDeviceMesh = PhysicalDeviceMesh
DistributedPhysicalDeviceMesh = PhysicalDeviceMesh


class VirtualPhysicalMesh:
    """A mesh description that holds no resources; sliced by the inter-op planner into submeshes
    (reference: device_mesh.py:1792-1976)."""

    def __init__(self, host_ids: Sequence[int], num_devices_per_host: int, devices: Optional[List[List[int]]] = None,
                 parent: Optional["VirtualPhysicalMesh"] = None, emulated: bool = False):
        self.host_ids = list(host_ids)
        self.num_devices_per_host = num_devices_per_host
        self.emulated = emulated
        if devices is None:
            devices = [[h * num_devices_per_host + i for i in range(num_devices_per_host)] for h in self.host_ids]
        self.devices = devices
        self.parent = parent
        self.launched_physical_mesh: Optional[PhysicalDeviceMesh] = None
        self.launched_physical_mesh_group: Optional["PhysicalDeviceMeshGroup"] = None

    @property
    def num_hosts(self):
        return len(self.host_ids)

    @property
    def shape(self):
        return (self.num_hosts, self.num_devices_per_host)

    @property
    def num_devices(self):
        return self.num_hosts * self.num_devices_per_host

    @property
    def flat_devices(self):
        return [d for row in self.devices for d in row]

    def slice_1d(self, dim: int, indices: Sequence[int]):
        if dim == 0:
            return VirtualPhysicalMesh([self.host_ids[i] for i in indices], self.num_devices_per_host,
                                       [self.devices[i] for i in indices], parent=self, emulated=self.emulated)
        assert dim == 1
        if indices and isinstance(indices[0], (list, tuple)):
            devs = [[row[i] for i in idx] for row, idx in zip(self.devices, indices)]
        else:
            devs = [[row[i] for i in indices] for row in self.devices]
        return VirtualPhysicalMesh(self.host_ids, len(devs[0]), devs, parent=self, emulated=self.emulated)

    def slice_2d(self, host_indices, device_indices):
        hosts = [self.host_ids[i] for i in host_indices]
        devs = [[self.devices[h][i] for i in device_indices[k]] for k, h in enumerate(host_indices)]
        return VirtualPhysicalMesh(hosts, len(devs[0]), devs, parent=self, emulated=self.emulated)

    def slice_profiling_submeshes(self, submesh_num_hosts, submesh_num_devices_per_host):
        """Tile the mesh with equal submeshes for stage profiling (reference :1903-1951)."""
        num_hosts, ndph = self.num_hosts, self.num_devices_per_host
        nh_chunks = num_hosts // submesh_num_hosts
        nd_chunks = ndph // submesh_num_devices_per_host
        out = []
        for i in range(nh_chunks):
            for j in range(nd_chunks):
                hi = list(range(i * submesh_num_hosts, (i + 1) * submesh_num_hosts))
                di = [list(range(j * submesh_num_devices_per_host, (j + 1) * submesh_num_devices_per_host))] * len(hi)
                out.append(self.slice_2d(hi, di))
        return out

    def get_logical_mesh(self, mesh_shape=None, mesh_alpha=None, mesh_beta=None):
        if mesh_shape is None:
            mesh_shape = self.shape
        id_mesh = np.array(self.flat_devices).reshape(tuple(mesh_shape))
        if mesh_alpha is None:
            mesh_alpha = (1,) * len(mesh_shape)
        if mesh_beta is None:
            mesh_beta = (1, 0.1) if self.num_hosts > 1 and len(mesh_shape) == 2 else (1,) * len(mesh_shape)
        return LogicalDeviceMesh(None, id_mesh, mesh_alpha, mesh_beta)

    def get_physical_mesh(self) -> PhysicalDeviceMesh:
        if self.launched_physical_mesh is None:
            self.launched_physical_mesh = PhysicalDeviceMesh(self.flat_devices, self.num_hosts,
                                                             emulated=self.emulated, parent=self)
        return self.launched_physical_mesh

    def get_physical_mesh_group(self, sliced_virtual_meshes: Sequence["VirtualPhysicalMesh"]):
        assert self.launched_physical_mesh_group is None or True
        meshes = [v.get_physical_mesh() for v in sliced_virtual_meshes]
        self.launched_physical_mesh_group = PhysicalDeviceMeshGroup(meshes, self)
        return self.launched_physical_mesh_group

    def __repr__(self):
        return f"VirtualPhysicalMesh(shape={self.shape}, devices={self.devices})"


class PhysicalDeviceMeshGroup:
    """The meshes of one pipeshard executable (reference: device_mesh.py:1979-2128)."""

    def __init__(self, meshes: List[PhysicalDeviceMesh], parent: Optional[VirtualPhysicalMesh]):
        self.meshes = list(meshes)
        self.parent = parent
        self.collective_groups: List[List[Any]] = [[None] * len(meshes) for _ in meshes]

    def __getitem__(self, i):
        return self.meshes[i]

    def __len__(self):
        return len(self.meshes)

    def index(self, m):
        return self.meshes.index(m)

    def my_mesh_index(self) -> Optional[int]:
        for i, m in enumerate(self.meshes):
            if m.is_member:
                return i
        return None

    def sync_workers(self):
        if dist.is_initialized():
            dist.barrier()

    def shutdown(self):
        for m in self.meshes:
            m.shutdown()

    def exception_shutdown(self):
        self.shutdown()

    # (reference: PhysicalDeviceMeshGroup, device_mesh.py:2040-2128)
    def set_runtime_random_seed(self, seed: int):
        for m in self.meshes:
            m.set_runtime_random_seed(seed)

    def sync_move_workers(self):
        for m in self.meshes:
            m.sync_move_workers()

    def get_memory_allocated(self):
        """Largest current allocation over the meshes this rank belongs to."""
        return max([m.get_memory_allocated() for m in self.meshes if m.is_member] or [0])

    def get_max_memory_allocated(self):
        return max([m.get_max_memory_allocated() for m in self.meshes if m.is_member] or [0])

    def get_max_memory_allocated_per_mesh(self):
        return [m.get_max_memory_allocated() if m.is_member else 0 for m in self.meshes]

    def reset_memory_stats(self):
        for m in self.meshes:
            if m.is_member:
                m.reset_memory_stats()

    def destroy_collective_groups(self):
        """(reference: tears down the cross-mesh NCCL groups; torch.distributed groups live until shutdown)"""
        self.collective_groups = [[None] * len(self.meshes) for _ in self.meshes]


class DeviceCluster:
    """All devices visible to the job (reference: device_mesh.py:2131-2305).

    With torchrun: world_size ranks, `devices_per_node` ranks per host.  With `cluster="local"`:
    `num_devices` emulated devices inside this process (1 by default)."""

    def __init__(self, num_nodes: Optional[int] = None, num_devices_per_node: Optional[int] = None,
                 emulated: bool = False):
        if emulated or not dist.is_initialized():
            self.num_hosts = num_nodes or 1
            self.num_devices_per_host = num_devices_per_node or 1
            self.emulated = True
        else:
            world = dist.get_world_size()
            local_world = int(os.environ.get("LOCAL_WORLD_SIZE", world))
            self.num_hosts = num_nodes or max(1, world // local_world)
            self.num_devices_per_host = num_devices_per_node or world // self.num_hosts
            self.emulated = False
        self.host_info = [{"NodeName": f"node{i}"} for i in range(self.num_hosts)]

    @property
    def num_devices(self):
        return self.num_hosts * self.num_devices_per_host

    @property
    def num_cpus(self):
        return os.cpu_count()

    def get_physical_mesh(self, host_ids=None, num_devices_per_host=None):
        host_ids = host_ids or list(range(self.num_hosts))
        n = num_devices_per_host or self.num_devices_per_host
        return self.get_virtual_physical_mesh(host_ids, n).get_physical_mesh()

    def get_virtual_physical_mesh(self, host_ids=None, num_devices_per_host=None):
        host_ids = host_ids or list(range(self.num_hosts))
        n = num_devices_per_host or self.num_devices_per_host
        devices = [[h * self.num_devices_per_host + i for i in range(n)] for h in host_ids]
        return VirtualPhysicalMesh(host_ids, n, devices, emulated=self.emulated)

    def profile_all(self, *args, **kwargs):
        from alpa_b200.mesh_profiling import profile_all
        return profile_all(self, *args, **kwargs)


########################################
# distributed arrays
########################################


# Live-array registry: which DistributedArrays still hold device memory on which mesh (reference: the worker-side
# buffer table behind MeshHostWorker.get_live_buffer_uuids, device_mesh.py:165-271, used by tests/runtime/
# test_memory_leak.py).  Weak references: an array leaves the table when it is deleted, donated or garbage collected.
_array_uuid = itertools.count(1)
_live_arrays: "weakref.WeakValueDictionary[int, DistributedArray]" = weakref.WeakValueDictionary()


def _register_live_array(arr: "DistributedArray"):
    _live_arrays[arr.uuid] = arr


def get_live_buffer_uuids(device_mesh: Optional["PhysicalDeviceMesh"] = None) -> List[int]:
    """uuids of the arrays that still own shards (optionally only those on `device_mesh`)."""
    out = []
    for uid, a in list(_live_arrays.items()):
        if a.deleted or not a.shards:
            continue
        if device_mesh is not None and tuple(a.device_mesh.devices) != tuple(device_mesh.devices):
            continue
        out.append(uid)
    return sorted(out)


def get_live_buffer_bytes(device_mesh: Optional["PhysicalDeviceMesh"] = None) -> int:
    """Bytes of shard storage (this process) still referenced by live arrays; shared storages are counted once."""
    seen, total = set(), 0
    ids = set(get_live_buffer_uuids(device_mesh))
    for uid, a in list(_live_arrays.items()):
        if uid not in ids:
            continue
        for t in a.shards:
            st = t.untyped_storage()
            key = (st.data_ptr(), st.nbytes())
            if key not in seen:
                seen.add(key)
                total += st.nbytes()
    return total


class DistributedArray:
    """A tensor tiled over a mesh; this process holds `shards` for its local devices.

    Reference: DistributedArray (device_mesh.py:1509-1694).  `_value` gathers the full array (all
    member ranks must call it, like any collective).  Donation = the executable reuses `shards`.
    """

    def __init__(self, device_mesh: PhysicalDeviceMesh, logical_mesh: LogicalDeviceMesh, shape, dtype,
                 sharding_spec: ShardingSpec, shards: List[torch.Tensor]):
        self.device_mesh = device_mesh
        self.logical_mesh = logical_mesh
        self.shape = tuple(shape)
        self.dtype = dtype
        self.sharding_spec = sharding_spec
        self.shards = shards
        self._full = None
        self.deleted = False
        self.uuid = next(_array_uuid)
        _register_live_array(self)

    @property
    def ndim(self):
        return len(self.shape)

    @property
    def size(self):
        return int(np.prod(self.shape)) if self.shape else 1

    @property
    def indices(self):
        return self.sharding_spec.indices(self.shape)

    @property
    def local_shard(self) -> torch.Tensor:
        assert not self.deleted, "array was donated/deleted"
        return self.shards[0]

    def delete(self):
        self.shards = []
        self._full = None
        self.deleted = True

    def is_deleted(self):
        return self.deleted

    def block_until_ready(self):
        if self.shards and self.shards[0].is_cuda:
            torch.cuda.synchronize()
        return self

    def full_tensor(self) -> torch.Tensor:
        """Gather the global value.  Collective: every rank of the job calls it (SPMD); members of the
        owning mesh gather the shards, and when the mesh is a strict subset of the world its first
        device broadcasts the result so that ranks of other pipeline stages see the same value."""
        assert not self.deleted, "array was donated/deleted"
        spec, lm, comm = self.sharding_spec, self.logical_mesh, self.device_mesh.comm
        full = None
        if self.device_mesh.is_member:
            xs = list(self.shards)
            for dim in range(len(self.shape)):
                for a in reversed(spec.dim_axes[dim]):
                    if lm.shape[a] > 1:
                        xs = comm.all_gather(xs, lm, a, dim)
            full = xs[0]
        if (not self.device_mesh.emulated and dist.is_initialized() and
                len(self.device_mesh.devices) < dist.get_world_size()):
            root = self.device_mesh.devices[0]
            if full is None:
                full = torch.empty(self.shape, dtype=self.dtype, device=self.device_mesh.torch_device)
            full = full.contiguous()
            dist.broadcast(full, src=root)
        return full

    @property
    def _value(self):
        if self._full is None:
            self._full = self.full_tensor().detach().cpu()
        return self._full

    def numpy(self):
        v = self._value
        return v.float().numpy() if v.dtype == torch.bfloat16 else v.numpy()

    # (reference: DistributedArray.prefetch / flush / to_np_async, device_mesh.py:1500-1560 -- asynchronous fetch of the
    # remote buffers to the driver.  Here the value is a collective gather; `prefetch` performs it once and caches it.)
    def prefetch(self):
        _ = self._value
        return self

    def flush(self):
        """Drop the cached host copy (the next `_value` gathers again)."""
        self._full = None

    def to_np_async(self):
        """Returns a zero-argument callable that yields the numpy value (reference: a future resolved by ray.get)."""
        self.prefetch()
        return self.numpy

    @property
    def one_replica_buffer_ids(self) -> List[int]:
        """Indices (into the mesh's device list) of one device per DISTINCT shard -- the shards a checkpoint has to
        write (reference: one_replica_buffer_ids, device_mesh.py:1462-1470)."""
        seen, out = set(), []
        for i, d in enumerate(self.logical_mesh.flatten_ids):
            key = tuple((sl.start, sl.stop) for sl in self.sharding_spec.local_slices(self.shape,
                                                                                     self.logical_mesh.coords_of(d)))
            if key not in seen:
                seen.add(key)
                out.append(i)
        return out

    def __array__(self, dtype=None):
        a = self.numpy()
        return a.astype(dtype) if dtype is not None else a

    def __float__(self):
        return float(self._value)

    def item(self):
        return self._value.item()

    def __repr__(self):
        return (f"DistributedArray(shape={self.shape}, dtype={self.dtype}, spec={self.sharding_spec}, "
                f"mesh={self.logical_mesh.shape})")

    # checkpoint hooks (format: alpa_b200/serialization.py)
    def save(self, path: str):
        from alpa_b200.serialization import save_distributed_array
        save_distributed_array(self, path)

    @classmethod
    def load(cls, path: str, aval_shape, dtype, device_mesh, logical_mesh, sharding_spec):
        from alpa_b200.serialization import load_distributed_array
        return load_distributed_array(path, aval_shape, dtype, device_mesh, logical_mesh, sharding_spec)


class ReplicatedDistributedArray:
    """The same logical array materialised on several meshes (reference: device_mesh.py:1697-1752)."""

    def __init__(self, device_meshes: Sequence[PhysicalDeviceMesh], arrays: Sequence[DistributedArray]):
        self._mesh_array_map = dict(zip(device_meshes, arrays))
        self.replica = arrays[0]
        self.shape = self.replica.shape
        self.dtype = self.replica.dtype

    def is_replicated_on_mesh(self, mesh):
        return mesh in self._mesh_array_map

    def get_replica_on_mesh(self, mesh):
        return self._mesh_array_map.get(mesh)

    def add_replica(self, mesh, array):
        self._mesh_array_map[mesh] = array

    @property
    def meshes(self):
        return list(self._mesh_array_map.keys())

    @property
    def _value(self):
        for m, a in self._mesh_array_map.items():
            if m.is_member:
                return a._value
        return self.replica._value

    def __array__(self, dtype=None):
        return np.asarray(self._value, dtype=dtype)


def prefetch(dis_arrays):
    """Start fetching the values of a pytree of DistributedArrays (reference :1755-1789).  With one
    process per GPU there is no RPC to overlap; we gather eagerly so later `_value` reads are free."""
    from torch.utils._pytree import tree_leaves
    for a in tree_leaves(dis_arrays):
        if isinstance(a, (DistributedArray, ReplicatedDistributedArray)):
            _ = a._value


########################################
# global runtime state
########################################
global_cluster: Optional[DeviceCluster] = None
global_physical_mesh: Optional[PhysicalDeviceMesh] = None
global_virtual_physical_mesh: Optional[VirtualPhysicalMesh] = None
_owns_process_group = False


def _default_torch_device() -> torch.device:
    if global_config.backend == "gpu" and torch.cuda.is_available():
        return torch.device("cuda", torch.cuda.current_device())
    return torch.device("cpu")


def init_global_cluster(cluster: str = "auto", cluster_address=None, num_nodes=None,
                        num_devices_per_node=None, namespace=None, num_devices=None, backend=None):
    """Reference: init_global_cluster (device_mesh.py:2314-2334).

    cluster = "local"        : this process only (optionally `num_devices` emulated devices)
              "distributed"  : torchrun-style env (RANK / WORLD_SIZE / MASTER_ADDR / MASTER_PORT)
              "auto" / "ray" : "distributed" if WORLD_SIZE>1 in the environment, else "local"
    """
    global global_cluster, global_physical_mesh, global_virtual_physical_mesh, _owns_process_group
    if backend is not None:
        global_config.backend = backend
    if not torch.cuda.is_available():
        global_config.backend = "cpu"
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if cluster in ("auto", "ray"):
        cluster = "distributed" if (world > 1 or dist.is_initialized()) else "local"
    if cluster == "local":
        n = num_devices or (num_devices_per_node or 1) * (num_nodes or 1)
        global_cluster = DeviceCluster(num_nodes or 1, n // (num_nodes or 1), emulated=True)
        global_virtual_physical_mesh = global_cluster.get_virtual_physical_mesh()
        global_physical_mesh = global_virtual_physical_mesh.get_physical_mesh()
    elif cluster == "distributed":
        if not dist.is_initialized():
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            os.environ.setdefault("MASTER_PORT", "29511")
            if global_config.backend == "gpu":
                torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
                dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
            else:
                dist.init_process_group("gloo")
            _owns_process_group = True
        global_cluster = DeviceCluster(num_nodes, num_devices_per_node)
        global_virtual_physical_mesh = global_cluster.get_virtual_physical_mesh()
        global_physical_mesh = None  # created lazily (reference keeps resources virtual until compile)
    else:
        raise ValueError(f"unknown cluster type {cluster!r}")


def shutdown_global_cluster():
    global global_cluster, global_physical_mesh, global_virtual_physical_mesh, _owns_process_group
    if global_physical_mesh is not None:
        global_physical_mesh.shutdown()
    global_cluster = global_physical_mesh = global_virtual_physical_mesh = None
    if _owns_process_group and dist.is_initialized():
        dist.destroy_process_group()
        DistCommunicator._group_cache.clear()
    _owns_process_group = False


def set_global_cluster(cluster: DeviceCluster):
    global global_cluster
    global_cluster = cluster


def get_global_cluster():
    return global_cluster


def set_global_physical_mesh(mesh: PhysicalDeviceMesh):
    global global_physical_mesh
    global_physical_mesh = mesh


def get_global_physical_mesh(create_if_not_exist=False):
    global global_physical_mesh
    if global_physical_mesh is None and create_if_not_exist:
        if global_virtual_physical_mesh is None:
            init_global_cluster("auto")
        global_physical_mesh = global_virtual_physical_mesh.get_physical_mesh()
    return global_physical_mesh


def set_global_virtual_physical_mesh(mesh: VirtualPhysicalMesh):
    global global_virtual_physical_mesh
    global_virtual_physical_mesh = mesh


def get_global_virtual_physical_mesh():
    return global_virtual_physical_mesh


def get_global_num_devices():
    if global_virtual_physical_mesh is not None:
        return global_virtual_physical_mesh.num_devices
    if global_physical_mesh is not None:
        return global_physical_mesh.num_devices
    raise RuntimeError("Please call alpa_b200.init first")
