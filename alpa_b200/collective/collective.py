"""Named collective groups and collective calls on plain tensors.

Reference: alpa/collective/collective.py (GroupManager:74, init_collective_group:151, create_collective_group:186,
allreduce:261 ... send:566, recv:629, _check_and_get_group:734) with NCCL/Gloo backends implemented on cupy / pygloo
(collective_group/*.py), stream pools (cuda_stream.py) and a Ray-actor rendezvous.

H100 design: one process per GPU already shares a `torch.distributed` world (NCCL over NVLink/NVSwitch; gloo on
CPU hosts), so a named group is a `dist.new_group` handle plus the rank translation table.  Rendezvous is the
world's store -- no actors.  P2P between two ranks uses batched isend/irecv (one NCCL group launch per direction,
like the reference's 2-rank communicators, without creating a communicator per GPU pair).  Collectives that have
a fused peer-memory implementation are in `alpa_b200.collective.fused`.
"""
from __future__ import annotations

import logging
from typing import Dict, List, Optional, Sequence

import torch
import torch.distributed as dist

logger = logging.getLogger(__name__)


class ReduceOp:
    SUM = "sum"
    PRODUCT = "product"
    MIN = "min"
    MAX = "max"


_TORCH_OP = {ReduceOp.SUM: dist.ReduceOp.SUM, ReduceOp.PRODUCT: dist.ReduceOp.PRODUCT,
             ReduceOp.MIN: dist.ReduceOp.MIN, ReduceOp.MAX: dist.ReduceOp.MAX}


class CollectiveGroup:
    def __init__(self, name: str, ranks: Sequence[int], backend: Optional[str], handle):
        self.name = name
        self.ranks = list(ranks)              # world ranks, position = rank inside the group
        self.backend = backend
        self.handle = handle

    @property
    def world_size(self):
        return len(self.ranks)

    def rank_of(self, world_rank: int) -> int:
        return self.ranks.index(world_rank) if world_rank in self.ranks else -1


class GroupManager:
    """Keeps the named groups of this process (reference: GroupManager, collective.py:74-148)."""

    def __init__(self):
        self._groups: Dict[str, CollectiveGroup] = {}

    def create_collective_group(self, backend: Optional[str], world_size: int, rank: int, group_name: str,
                                ranks: Optional[Sequence[int]] = None, store=None) -> CollectiveGroup:
        if backend == "native":
            # communicators, streams and events owned by the C++ module (csrc/comm_group.cpp); only the members take
            # part in the creation (reference: the NCCL groups of collective_group/nccl_collective_group.py, which are
            # likewise independent of any global process group)
            from alpa_b200.collective.native_group import NativeCommGroup
            from alpa_b200.global_env import global_config
            ranks = list(ranks) if ranks is not None else list(range(world_size))
            assert len(ranks) == world_size and ranks == sorted(ranks), "native groups order their members by world rank"
            kw = {"backend": global_config.native_comm_backend} if global_config.native_comm_backend is not None else {}
            g = CollectiveGroup(group_name, ranks, "native", NativeCommGroup(ranks, ranks[rank], store=store, **kw))
            g.my_rank = ranks[rank]
            self._groups[group_name] = g
            return g
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed is not initialised: call alpa_b200.init(cluster='distributed') "
                               "or dist.init_process_group first")
        ranks = list(ranks) if ranks is not None else list(range(world_size))
        assert len(ranks) == world_size
        # every process of the world must call new_group, in the same order
        handle = dist.new_group(ranks=ranks, backend=backend)
        g = CollectiveGroup(group_name, ranks, backend, handle)
        self._groups[group_name] = g
        return g

    def is_group_exist(self, group_name: str) -> bool:
        return group_name in self._groups

    def get_group_by_name(self, group_name: str) -> CollectiveGroup:
        if group_name not in self._groups:
            raise KeyError(f"The collective group '{group_name}' is not initialized")
        return self._groups[group_name]

    def destroy_collective_group(self, group_name: str):
        g = self._groups.pop(group_name, None)
        if g is not None and g.backend == "native":
            g.handle.destroy()
            return
        if g is not None and g.handle is not None:
            try:
                dist.destroy_process_group(g.handle)
            except Exception as e:  # noqa: BLE001
                logger.debug("destroy group %s: %s", group_name, e)


_group_mgr = GroupManager()


def is_group_initialized(group_name: str) -> bool:
    return _group_mgr.is_group_exist(group_name)


def init_collective_group(world_size: int, rank: int, backend: Optional[str] = None, group_name: str = "default",
                          ranks: Optional[Sequence[int]] = None, store=None):
    """Create the named group in this process (collective over the whole world; reference: collective.py:151).
    backend: None / "nccl" / "gloo" = torch.distributed groups; "native" = the C++ communication groups (collective over
    the members only; `store` = the key-value store of the id exchange, default the torch.distributed store)."""
    if _group_mgr.is_group_exist(group_name):
        raise RuntimeError(f"Trying to initialize a group twice: {group_name}")
    assert world_size > 0 and 0 <= rank < world_size
    return _group_mgr.create_collective_group(backend, world_size, rank, group_name, ranks, store)


class _NativeOps:
    """The named-group operations on a native group: issued on the group's own streams, bracketed so that the call
    keeps the stream-ordered semantics of the torch.distributed path (inputs produced on the current stream are
    complete before the transfer, the result is visible to the current stream afterwards)."""

    def __init__(self, g: CollectiveGroup):
        self.g, self.n = g, g.handle

    def __enter__(self):
        self.n.comm_wait_compute()
        return self.n

    def __exit__(self, *exc):
        self.n.compute_wait_comm()
        return False


def create_collective_group(ranks: Sequence[int], backend: Optional[str] = None, group_name: str = "default"):
    """Declarative form: the group of the given world ranks (reference: create_collective_group, collective.py:186,
    which takes actor handles)."""
    me = dist.get_rank()
    return init_collective_group(len(ranks), ranks.index(me) if me in ranks else 0, backend, group_name, ranks)


def _me(g: Optional[CollectiveGroup] = None) -> int:
    """This process's world rank (a native group remembers it: it does not need an initialised process group)."""
    r = getattr(g, "my_rank", None) if g is not None else None
    return r if r is not None else dist.get_rank()


def destroy_collective_group(group_name: str = "default"):
    _group_mgr.destroy_collective_group(group_name)


def get_rank(group_name: str = "default") -> int:
    if not is_group_initialized(group_name):
        return -1
    g = _group_mgr.get_group_by_name(group_name)
    return g.rank_of(_me(g))


def get_collective_group_size(group_name: str = "default") -> int:
    if not is_group_initialized(group_name):
        return -1
    return _group_mgr.get_group_by_name(group_name).world_size


def _check_and_get_group(group_name: str) -> CollectiveGroup:
    return _group_mgr.get_group_by_name(group_name)


def allreduce(tensor: torch.Tensor, group_name: str = "default", op: str = ReduceOp.SUM):
    g = _check_and_get_group(group_name)
    if g.backend == "native":
        with _NativeOps(g) as n:
            n.all_reduce(tensor, {ReduceOp.SUM: "sum", ReduceOp.PRODUCT: "prod", ReduceOp.MIN: "min",
                                  ReduceOp.MAX: "max"}[op])
        return tensor
    dist.all_reduce(tensor, op=_TORCH_OP[op], group=g.handle)
    return tensor


def barrier(group_name: str = "default"):
    g = _check_and_get_group(group_name)
    if g.backend == "native":
        allreduce(torch.zeros(1, device="cuda" if torch.cuda.is_available() else "cpu"), group_name)
        g.handle.synchronize()
        return
    dist.barrier(group=_check_and_get_group(group_name).handle)


def reduce(tensor: torch.Tensor, dst_rank: int = 0, group_name: str = "default", op: str = ReduceOp.SUM):
    g = _check_and_get_group(group_name)
    if g.backend == "native":                     # every member ends up with the result; the destination asked for it
        return allreduce(tensor, group_name, op)
    dist.reduce(tensor, dst=g.ranks[dst_rank], op=_TORCH_OP[op], group=g.handle)
    return tensor


def broadcast(tensor: torch.Tensor, src_rank: int = 0, group_name: str = "default"):
    g = _check_and_get_group(group_name)
    if g.backend == "native":
        with _NativeOps(g) as n:
            n.broadcast(tensor, g.ranks[src_rank])
        return tensor
    dist.broadcast(tensor, src=g.ranks[src_rank], group=g.handle)
    return tensor


def allgather(tensor_list: List[torch.Tensor], tensor: torch.Tensor, group_name: str = "default"):
    g = _check_and_get_group(group_name)
    assert len(tensor_list) == g.world_size
    if g.backend == "native":
        out = torch.empty((g.world_size,) + tuple(tensor.shape), dtype=tensor.dtype, device=tensor.device)
        with _NativeOps(g) as n:
            n.all_gather(out, tensor.contiguous())
        for t, o in zip(tensor_list, out):
            t.copy_(o)
        return tensor_list
    dist.all_gather(tensor_list, tensor, group=g.handle)
    return tensor_list


def reducescatter(tensor: torch.Tensor, tensor_list: List[torch.Tensor], group_name: str = "default",
                  op: str = ReduceOp.SUM):
    g = _check_and_get_group(group_name)
    assert len(tensor_list) == g.world_size
    if g.backend == "native":
        with _NativeOps(g) as n:
            n.reduce_scatter(tensor, torch.stack(list(tensor_list)), {ReduceOp.SUM: "sum", ReduceOp.PRODUCT: "prod",
                                                                       ReduceOp.MIN: "min", ReduceOp.MAX: "max"}[op])
        return tensor
    if g.backend == "gloo" or (g.backend is None and dist.get_backend() == "gloo"):
        # gloo has no reduce_scatter: all-reduce the concatenation and keep our part
        cat = torch.stack(list(tensor_list))
        dist.all_reduce(cat, op=_TORCH_OP[op], group=g.handle)
        tensor.copy_(cat[g.rank_of(dist.get_rank())])
    else:
        dist.reduce_scatter(tensor, list(tensor_list), op=_TORCH_OP[op], group=g.handle)
    return tensor


def send(tensor: torch.Tensor, dst_rank: int, group_name: str = "default"):
    g = _check_and_get_group(group_name)
    if g.ranks[dst_rank] == _me(g):
        raise RuntimeError(f"The destination rank '{dst_rank}' is self.")
    if g.backend == "native":
        with _NativeOps(g) as n:
            n.send(tensor.contiguous(), g.ranks[dst_rank])
        return
    dist.send(tensor, dst=g.ranks[dst_rank], group=g.handle)


def recv(tensor: torch.Tensor, src_rank: int, group_name: str = "default"):
    g = _check_and_get_group(group_name)
    if g.ranks[src_rank] == _me(g):
        raise RuntimeError(f"The source rank '{src_rank}' is self.")
    if g.backend == "native":
        with _NativeOps(g) as n:
            n.recv(tensor, g.ranks[src_rank])
        return tensor
    dist.recv(tensor, src=g.ranks[src_rank], group=g.handle)
    return tensor


def batch_send_recv(sends: Sequence, recvs: Sequence, group_name: str = "default"):
    """One grouped launch for many tile transfers: sends = [(tensor, dst_rank)], recvs = [(tensor, src_rank)]
    (the cross-mesh resharding path; reference: NCCLGroup.send_multigpu/recv_multigpu pairs)."""
    g = _check_and_get_group(group_name)
    if g.backend == "native":
        with _NativeOps(g) as n:
            n.batch([("send", t, g.ranks[r], -1, -1) for t, r in sends] +
                    [("recv", t, g.ranks[r], -1, -1) for t, r in recvs])
        return
    ops = [dist.P2POp(dist.isend, t, g.ranks[r], g.handle) for t, r in sends]
    ops += [dist.P2POp(dist.irecv, t, g.ranks[r], g.handle) for t, r in recvs]
    if not ops:
        return
    for w in dist.batch_isend_irecv(ops):
        w.wait()


def synchronize(gpu_id: Optional[int] = None):
    if torch.cuda.is_available():
        torch.cuda.synchronize(gpu_id)


# ------------------------------------------------------------------------------------------------
# the rest of the reference's module surface (alpa/collective/collective.py)
# ------------------------------------------------------------------------------------------------
def nccl_available() -> bool:
    return dist.is_available() and dist.is_nccl_available() and torch.cuda.is_available()


def gloo_available() -> bool:
    return dist.is_available() and dist.is_gloo_available()


def get_nccl_group(world_size: int, rank: int, group_name: str = "default"):
    """(reference: get_nccl_group) -- the named group, created on first use."""
    if not is_group_initialized(group_name):
        init_collective_group(world_size, rank, "nccl" if nccl_available() else "gloo", group_name)
    return _check_and_get_group(group_name)


# One process drives one GPU here, so the reference's *_multigpu variants (one process driving several GPUs with a
# tensor per GPU) reduce to the single-tensor collectives over a one-element list.
def allreduce_multigpu(tensor_list, group_name: str = "default", op: str = ReduceOp.SUM):
    assert len(tensor_list) == 1, "one process drives one GPU"
    return [allreduce(tensor_list[0], group_name, op)]


def reduce_multigpu(tensor_list, dst_rank: int = 0, dst_tensor: int = 0, group_name: str = "default",
                    op: str = ReduceOp.SUM):
    assert len(tensor_list) == 1 and dst_tensor == 0
    return [reduce(tensor_list[0], dst_rank, group_name, op)]


def broadcast_multigpu(tensor_list, src_rank: int = 0, src_tensor: int = 0, group_name: str = "default"):
    assert len(tensor_list) == 1 and src_tensor == 0
    return [broadcast(tensor_list[0], src_rank, group_name)]


def broadcast_partialgpu(tensor_list, n_elements, comm_key, world_size, devices_ids, devices_global_rank,
                         group_name: str = "default", local_start_pos_list=None):
    """Broadcast the first `n_elements` elements from the first listed rank (reference: broadcast_partialgpu, the
    cross-mesh broadcast resharding primitive)."""
    assert len(tensor_list) == 1
    t = tensor_list[0].reshape(-1)[:n_elements]
    buf = t.contiguous()
    broadcast(buf, devices_global_rank[0], group_name)
    if buf.data_ptr() != t.data_ptr():
        t.copy_(buf)
    return tensor_list


def allgather_multigpu(output_tensor_lists, input_tensor_list, group_name: str = "default"):
    assert len(input_tensor_list) == 1 and len(output_tensor_lists) == 1
    return [allgather(output_tensor_lists[0], input_tensor_list[0], group_name)]


def reducescatter_multigpu(output_tensor_list, input_tensor_lists, group_name: str = "default", op: str = ReduceOp.SUM):
    assert len(output_tensor_list) == 1 and len(input_tensor_lists) == 1
    return [reducescatter(output_tensor_list[0], input_tensor_lists[0], group_name, op)]


def send_multigpu(tensor, dst_rank: int, dst_gpu_index: int = 0, group_name: str = "default", start_pos=None,
                  n_elements=None):
    t = tensor if n_elements is None else tensor.reshape(-1)[(start_pos or 0):(start_pos or 0) + n_elements]
    return send(t.contiguous(), dst_rank, group_name)


def recv_multigpu(tensor, src_rank: int, src_gpu_index: int = 0, group_name: str = "default", start_pos=None,
                  n_elements=None):
    if n_elements is None:
        return recv(tensor, src_rank, group_name)
    flat = tensor.reshape(-1)
    buf = torch.empty(n_elements, dtype=tensor.dtype, device=tensor.device)
    recv(buf, src_rank, group_name)
    flat[(start_pos or 0):(start_pos or 0) + n_elements].copy_(buf)
    return tensor


# stream / event synchronisation between compute and communication (reference: record_events, wait_events,
# comm_wait_compute, compute_wait_comm -- XLA/service/gpu/alpa_events.cc through the group object)
from alpa_b200.collective.streams import (comm_wait_compute, compute_wait_comm, record_events,  # noqa: E402,F401
                                          wait_events)
