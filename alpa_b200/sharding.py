"""Sharding specs and the logical device mesh with its alpha-beta communication cost model.

``ShardingSpec`` plays the role of ``pxla.ShardingSpec``/``HloSharding`` in the reference
(alpa/shard_parallel/auto_sharding.py:81-169, 561-614): for every tensor dimension it records which
logical-mesh axes tile that dimension; axes that tile nothing replicate the tensor.

On a single NVSwitch domain both mesh axes have the same bandwidth; the defaults below are therefore
uniform, and `DeviceMesh.get_logical_mesh` can overwrite them with profiled values.
"""
from __future__ import annotations

import itertools
from dataclasses import dataclass
from typing import List, Sequence, Tuple

import numpy as np


@dataclass(frozen=True)
class ShardingSpec:
    """Tile-sharding of a tensor over a logical mesh.

    dim_axes[i] is the tuple of mesh axes (major to minor) that tile tensor dim i; () = not sharded.
    Each mesh axis appears at most once over the whole spec.
    """
    mesh_shape: Tuple[int, ...]
    dim_axes: Tuple[Tuple[int, ...], ...]

    # ---------------- constructors ----------------
    @staticmethod
    def replicated(mesh_shape: Sequence[int], ndim: int) -> "ShardingSpec":
        return ShardingSpec(tuple(mesh_shape), tuple(() for _ in range(ndim)))

    @staticmethod
    def from_dim_map(mesh_shape: Sequence[int], ndim: int, tensor_dims: Sequence[int],
                     mesh_dims: Sequence[int]) -> "ShardingSpec":
        """`tensor_dims[i]` is tiled along `mesh_dims[i]` (cf. LogicalDeviceMesh.make_tile_spec)."""
        axes: List[List[int]] = [[] for _ in range(ndim)]
        for t, m in zip(tensor_dims, mesh_dims):
            axes[t].append(m)
        return ShardingSpec(tuple(mesh_shape), tuple(tuple(a) for a in axes))

    @staticmethod
    def from_string(mesh_shape: Sequence[int], s: str) -> "ShardingSpec":
        """Parse the compact notation used in plans/tests: 'S0R', 'RS1', 'S01R', 'RR'."""
        dims = []
        i = 0
        while i < len(s):
            if s[i] == "R":
                dims.append(())
                i += 1
            elif s[i] == "S":
                j = i + 1
                while j < len(s) and s[j].isdigit():
                    j += 1
                dims.append(tuple(int(c) for c in s[i + 1:j]))
                i = j
            else:
                raise ValueError(f"bad sharding string {s!r}")
        return ShardingSpec(tuple(mesh_shape), tuple(dims))

    # ---------------- queries ----------------
    def __post_init__(self):
        used = [a for axes in self.dim_axes for a in axes]
        assert len(used) == len(set(used)), f"mesh axis used twice in {self.dim_axes}"
        assert all(0 <= a < len(self.mesh_shape) for a in used)

    @property
    def ndim(self) -> int:
        return len(self.dim_axes)

    def num_shards(self, dim: int) -> int:
        n = 1
        for a in self.dim_axes[dim]:
            n *= self.mesh_shape[a]
        return n

    def total_shards(self) -> int:
        return int(np.prod([self.num_shards(d) for d in range(self.ndim)])) if self.ndim else 1

    def used_axes(self) -> Tuple[int, ...]:
        return tuple(a for axes in self.dim_axes for a in axes if self.mesh_shape[a] > 1)

    def replicated_axes(self) -> Tuple[int, ...]:
        used = {a for axes in self.dim_axes for a in axes}
        return tuple(a for a in range(len(self.mesh_shape)) if a not in used and self.mesh_shape[a] > 1)

    def is_replicated(self) -> bool:
        return all(self.num_shards(d) == 1 for d in range(self.ndim))

    def shard_shape(self, global_shape: Sequence[int]) -> Tuple[int, ...]:
        out = []
        for d, g in enumerate(global_shape):
            n = self.num_shards(d)
            assert g % n == 0, f"dim {d} of size {g} not divisible into {n} shards"
            out.append(g // n)
        return tuple(out)

    def shard_index(self, dim: int, mesh_coords: Sequence[int]) -> int:
        idx = 0
        for a in self.dim_axes[dim]:
            idx = idx * self.mesh_shape[a] + mesh_coords[a]
        return idx

    def local_slices(self, global_shape: Sequence[int], mesh_coords: Sequence[int]) -> Tuple[slice, ...]:
        """The index (tuple of slices) of the shard held by the device at `mesh_coords`."""
        out = []
        for d, g in enumerate(global_shape):
            n = self.num_shards(d)
            size = g // n
            i = self.shard_index(d, mesh_coords)
            out.append(slice(i * size, (i + 1) * size))
        return tuple(out)

    def indices(self, global_shape: Sequence[int]) -> List[Tuple[slice, ...]]:
        """Shard index for every device in row-major logical-mesh order (cf. spec.indices(shape))."""
        return [self.local_slices(global_shape, c)
                for c in itertools.product(*[range(s) for s in self.mesh_shape])]

    def normalized(self) -> "ShardingSpec":
        """Drop mesh axes of size 1 (they never change the tiling)."""
        return ShardingSpec(self.mesh_shape,
                            tuple(tuple(a for a in axes if self.mesh_shape[a] > 1) for axes in self.dim_axes))

    def equivalent(self, other: "ShardingSpec") -> bool:
        return self.mesh_shape == other.mesh_shape and self.normalized().dim_axes == other.normalized().dim_axes

    def with_dim(self, dim: int, axes: Sequence[int]) -> "ShardingSpec":
        d = list(self.dim_axes)
        d[dim] = tuple(axes)
        return ShardingSpec(self.mesh_shape, tuple(d))

    def __str__(self) -> str:
        if self.ndim == 0:
            return "R"
        return "".join("R" if not axes else "S" + "".join(str(a) for a in axes) for axes in self.dim_axes)

    __repr__ = __str__


class LogicalDeviceMesh:
    """A logical 1-D/2-D view of a physical mesh with an alpha-beta cost model per mesh axis.

    Mirrors the interface of the reference class (auto_sharding.py:81-169).  Cost formulas keep the
    reference's structure (so closed-form plan costs in tests carry over) but the default betas are
    equal: through NVSwitch every peer is reachable at full NVLink 4 bandwidth.
    """

    def __init__(self, physical_mesh, id_mesh, mesh_alpha=None, mesh_beta=None):
        self.physical_mesh = physical_mesh
        self.id_mesh = np.array(id_mesh)
        self.flatten_ids = tuple(int(x) for x in self.id_mesh.flatten())
        nd = len(self.id_mesh.shape)
        self.mesh_alpha = tuple(mesh_alpha) if mesh_alpha is not None else (1,) * nd
        self.mesh_beta = tuple(mesh_beta) if mesh_beta is not None else (1,) * nd

    @property
    def shape(self):
        return tuple(int(s) for s in self.id_mesh.shape)

    @property
    def num_devices(self):
        return int(np.prod(self.id_mesh.shape))

    def flatten(self):
        """An effective 1-D mesh over the same devices (reference :114-121)."""
        return LogicalDeviceMesh(self.physical_mesh, self.id_mesh.reshape(-1, 1),
                                 [max(self.mesh_alpha)] * 2, [min(self.mesh_beta)] * 2)

    def all_gather_cost(self, num_bytes, mesh_dim):
        n = self.id_mesh.shape[mesh_dim]
        return self.mesh_alpha[mesh_dim] + self.mesh_beta[mesh_dim] * (n - 1) / n * num_bytes + 0.1

    def all_reduce_cost(self, num_bytes, mesh_dim):
        n = self.id_mesh.shape[mesh_dim]
        return self.mesh_alpha[mesh_dim] + self.mesh_beta[mesh_dim] * 2 * (n - 1) / n * num_bytes + 0.01

    def reduce_scatter_cost(self, num_bytes, mesh_dim):
        n = self.id_mesh.shape[mesh_dim]
        return self.mesh_alpha[mesh_dim] + self.mesh_beta[mesh_dim] * (n - 1) / n * num_bytes + 0.001

    def all_to_all_cost(self, num_bytes, mesh_dim):
        # Every device exchanges (n-1)/n of its 1/n shard.  The reference multiplies this by n/2 (ring-connected
        # V100s, auto_sharding.py:137-141); behind an NVSwitch every pair has a full-rate path, so no penalty.
        n = self.id_mesh.shape[mesh_dim]
        return self.mesh_alpha[mesh_dim] + self.mesh_beta[mesh_dim] * (n - 1) / n / n * num_bytes + 0.001

    def make_tile_spec(self, array_or_ndim, tensor_dims, mesh_dims) -> ShardingSpec:
        ndim = array_or_ndim if isinstance(array_or_ndim, int) else len(array_or_ndim.shape)
        return ShardingSpec.from_dim_map(self.shape, ndim, tensor_dims, mesh_dims)

    def coords_of(self, device_id: int) -> Tuple[int, ...]:
        pos = np.argwhere(self.id_mesh == device_id)
        assert len(pos) == 1, f"device {device_id} not in mesh {self.flatten_ids}"
        return tuple(int(x) for x in pos[0])

    def axis_group(self, device_id: int, mesh_dim: int) -> Tuple[int, ...]:
        """Device ids that differ from `device_id` only along `mesh_dim` (a collective group)."""
        c = list(self.coords_of(device_id))
        out = []
        for i in range(self.id_mesh.shape[mesh_dim]):
            c[mesh_dim] = i
            out.append(int(self.id_mesh[tuple(c)]))
        return tuple(out)

    def __hash__(self):
        return hash((self.flatten_ids, self.shape, self.mesh_alpha, self.mesh_beta))

    def __eq__(self, other):
        return (isinstance(other, LogicalDeviceMesh) and
                (self.flatten_ids, self.shape, self.mesh_alpha, self.mesh_beta) ==
                (other.flatten_ids, other.shape, other.mesh_alpha, other.mesh_beta))

    def __repr__(self):
        return f"LogicalDeviceMesh(shape={self.shape}, alpha={self.mesh_alpha}, beta={self.mesh_beta})"
