"""Input pipelines that hand the executables ready-sharded `DistributedArray`s.

Reference: alpa/data_loader.py (DataLoader:15 -- driver-side iterator with a prefetch queue that shards every
batch according to the executable's input placement specs; MeshDriverDataLoader:97 / MeshWorkerDataLoader:229 --
every host loads only the slice of the global batch that its own devices need).

H100 design: one process per GPU, so "each host loads its slice" becomes "each rank reads the rows its device's
shard covers".  Batches are staged in pinned host memory and copied on a dedicated CUDA copy stream, `prefetch_size`
batches ahead, so the H2D copy of step i+1 overlaps the compute of step i; consumers wait on the copy event only.
"""
from __future__ import annotations

import collections
import itertools
from typing import Callable, Iterable, Iterator, Optional

import numpy as np
import torch
import torch.utils._pytree as pytree

from alpa_b200 import device_mesh as dm
from alpa_b200.device_mesh import DistributedArray, PhysicalDeviceMesh
from alpa_b200.parallel_plan import PlacementSpec


def _resolve_mesh(spec: PlacementSpec, physical_mesh: Optional[PhysicalDeviceMesh]):
    mesh = physical_mesh or dm.get_global_physical_mesh(create_if_not_exist=True)
    want = tuple(spec.mesh_ids[0])
    if tuple(mesh.devices) != want:
        sub = getattr(mesh, "submesh_of_devices", None)
        mesh = sub(want) if sub is not None else mesh
    sspec = spec.sharding_specs[0]
    return mesh, mesh.get_logical_mesh(tuple(sspec.mesh_shape)), sspec


def _to_tensor(x) -> torch.Tensor:
    if isinstance(x, torch.Tensor):
        return x
    return torch.from_numpy(np.ascontiguousarray(x))


class _CopyPipe:
    """Pinned staging + copy stream shared by the loaders."""

    def __init__(self, device: torch.device):
        self.device = device
        self.cuda = device.type == "cuda"
        self.stream = torch.cuda.Stream(device=device) if self.cuda else None

    def put(self, host: torch.Tensor) -> torch.Tensor:
        if not self.cuda:
            return host.clone()
        if not host.is_pinned():
            host = host.pin_memory()
        with torch.cuda.stream(self.stream):
            dev = host.to(self.device, non_blocking=True)
        dev.record_stream(torch.cuda.current_stream(self.device))
        return dev

    def ready(self):
        if self.cuda:
            torch.cuda.current_stream(self.device).wait_stream(self.stream)


class DataLoader:
    """Iterate `input_iter` (pytrees of global numpy / torch batches), shard every leaf according to
    `placement_specs` (a pytree prefix or flat list of PlacementSpec) and keep `prefetch_size` batches in flight."""

    def __init__(self, input_iter: Iterable, placement_specs, prefetch_size: int = 1,
                 physical_mesh: Optional[PhysicalDeviceMesh] = None):
        self.input_iter = input_iter
        self.placement_specs = placement_specs
        self.prefetch_size = max(1, prefetch_size)
        self.physical_mesh = physical_mesh
        self._pipe = None
        self.queue: collections.deque = collections.deque()
        self.first_iter = True

    def _shard_batch(self, batch):
        leaves, tree = pytree.tree_flatten(batch)
        specs, _ = pytree.tree_flatten(self.placement_specs, is_leaf=lambda x: isinstance(x, PlacementSpec) or x is None)
        assert len(specs) == len(leaves), f"{len(specs)} placement specs for {len(leaves)} batch leaves"
        out = []
        for leaf, ps in zip(leaves, specs):
            if ps is None:
                out.append(leaf)
                continue
            mesh, lmesh, sspec = _resolve_mesh(ps, self.physical_mesh)
            if self._pipe is None:
                self._pipe = _CopyPipe(mesh.torch_device)
            t = _to_tensor(leaf)
            shards = []
            for d in mesh.local_devices:
                sl = sspec.local_slices(t.shape, lmesh.coords_of(d))
                shards.append(self._pipe.put(t[sl].contiguous()))
            out.append(DistributedArray(mesh, lmesh, tuple(t.shape), t.dtype, sspec, shards))
        return pytree.tree_unflatten(out, tree)

    def enqueue(self, num_batches: int):
        for batch in itertools.islice(self.input_iter, num_batches):
            self.queue.append(self._shard_batch(batch))

    def __iter__(self) -> Iterator:
        if self.first_iter:
            self.first_iter = False
            self.input_iter = iter(self.input_iter)
            self.enqueue(self.prefetch_size)
        while self.queue:
            item = self.queue.popleft()
            if self._pipe is not None:
                self._pipe.ready()
            self.enqueue(1)
            yield item


class MeshDriverDataLoader:
    """Every rank loads only the rows of the batch dim that its devices own.

    input_iter_func(start, end, batch_size) -> iterator over pytrees whose leaves have `end - start` rows: the
    rows [start, end) of every global batch (reference: MeshDriverDataLoader, data_loader.py:97-226; the worker
    half lives in the same class because every rank is both driver and worker here)."""

    def __init__(self, batch_size: int, num_samples: int, input_iter_func: Callable[[int, int, int], Iterable],
                 placement_specs, prefetch_size: int = 1, repeat: bool = False,
                 physical_mesh: Optional[PhysicalDeviceMesh] = None):
        self.batch_size = batch_size
        self.num_samples = num_samples
        self.steps_per_epoch = num_samples // batch_size
        self.input_iter_func = input_iter_func
        self.prefetch_size = max(1, prefetch_size)
        self.repeat = repeat
        self.physical_mesh = physical_mesh
        self.specs, self.spec_tree = pytree.tree_flatten(
            placement_specs, is_leaf=lambda x: isinstance(x, PlacementSpec) or x is None)
        # per leaf and local device: the row range of the batch dim it needs
        self.meshes = [None if s is None else _resolve_mesh(s, physical_mesh) for s in self.specs]
        lo, hi = batch_size, 0
        for s, m in zip(self.specs, self.meshes):
            if s is None:
                continue
            mesh, lmesh, sspec = m
            shape = tuple(s.aval[0]) if s.aval is not None else (batch_size,)
            for d in mesh.local_devices:
                sl = sspec.local_slices(shape, lmesh.coords_of(d))[0]
                lo, hi = min(lo, sl.start or 0), max(hi, sl.stop if sl.stop is not None else batch_size)
        self.row_range = (lo, hi) if hi > lo else (0, batch_size)
        self._pipe = None
        self.queue: collections.deque = collections.deque()
        self._iter = None

    def _make_iter(self):
        lo, hi = self.row_range
        it = iter(self.input_iter_func(lo, hi, self.batch_size))
        return itertools.cycle(it) if self.repeat else it

    def _shard_local(self, batch):
        leaves, tree = pytree.tree_flatten(batch)
        assert len(leaves) == len(self.specs)
        lo, _ = self.row_range
        out = []
        for leaf, s, m in zip(leaves, self.specs, self.meshes):
            if s is None:
                out.append(leaf)
                continue
            mesh, lmesh, sspec = m
            if self._pipe is None:
                self._pipe = _CopyPipe(mesh.torch_device)
            t = _to_tensor(leaf)
            gshape = (self.batch_size,) + tuple(t.shape[1:])
            shards = []
            for d in mesh.local_devices:
                sl = list(sspec.local_slices(gshape, lmesh.coords_of(d)))
                b = sl[0]
                sl[0] = slice((b.start or 0) - lo, (b.stop if b.stop is not None else self.batch_size) - lo)
                shards.append(self._pipe.put(t[tuple(sl)].contiguous()))
            out.append(DistributedArray(mesh, lmesh, gshape, t.dtype, sspec, shards))
        return pytree.tree_unflatten(out, tree)

    def _enqueue(self, n):
        for batch in itertools.islice(self._iter, n):
            self.queue.append(self._shard_local(batch))

    def __iter__(self):
        self._iter = self._make_iter()
        self.queue.clear()
        self._enqueue(self.prefetch_size)
        while self.queue:
            item = self.queue.popleft()
            if self._pipe is not None:
                self._pipe.ready()
            self._enqueue(1)
            yield item

    def __len__(self):
        return self.steps_per_epoch


# ---- helpers of the reference's module (alpa/data_loader.py)
import itertools as _itertools

_mesh_data_loader_counter = _itertools.count()


def next_mesh_data_loader_uuid() -> int:
    """(reference: data_loader.next_mesh_data_loader_uuid)"""
    return next(_mesh_data_loader_counter)


def get_num_devices_for_whole_batch(sharding_spec, batch_dim: int = 0) -> int:
    """How many consecutive devices of the mesh hold one whole batch: the product of the mesh axes that do NOT shard
    the batch dimension (reference: data_loader.get_num_devices_for_whole_batch, used to decide which hosts load which
    slice of the global batch)."""
    n = 1
    used = set(sharding_spec.dim_axes[batch_dim]) if batch_dim < len(sharding_spec.dim_axes) else set()
    for axis, size in enumerate(sharding_spec.mesh_shape):
        if axis not in used:
            n *= int(size)
    return n


MeshWorkerDataLoader = MeshDriverDataLoader      # one process per GPU: the driver-side loader IS the worker-side loader
