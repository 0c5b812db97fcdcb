"""Top-level user API: init / shutdown / parallelize / grad / value_and_grad.

Reference: alpa/api.py (init:25, shutdown:63, parallelize:71, ParallelizedFunc:106, grad:241,
value_and_grad:265).  The decorated function is ordinary PyTorch code over pytrees of tensors; it is
traced once per input signature into a flat graph (forward + backward + optimizer), planned, lowered
to a per-rank SPMD program of sm_90a kernels + collectives, and cached.
"""
from __future__ import annotations

import functools
from typing import Callable, Optional, Sequence, Union

import numpy as np
import torch
from torch.utils import _pytree as pytree

from alpa_b200 import device_mesh as dm
from alpa_b200.device_mesh import DistributedArray, ReplicatedDistributedArray
from alpa_b200.global_env import global_config

is_initialized = False


def init(cluster: str = "auto", cluster_address: Optional[str] = None, num_nodes: Optional[int] = None,
         num_devices_per_node: Optional[int] = None, namespace: Optional[str] = "alpa_default_space",
         num_devices: Optional[int] = None, backend: Optional[str] = None):
    """Initialise the global runtime (reference: alpa.init, api.py:25-60).

    cluster: "auto"/"ray" (torchrun world if WORLD_SIZE>1 else local), "local", "distributed".
    `num_devices` > 1 with cluster="local" creates an in-process emulated mesh (device-free testing)."""
    global is_initialized
    if is_initialized:
        return
    dm.init_global_cluster(cluster, cluster_address, num_nodes, num_devices_per_node, namespace,
                           num_devices=num_devices, backend=backend)
    is_initialized = True


def shutdown():
    """Release the runtime (reference: alpa.shutdown, api.py:63-68)."""
    global is_initialized
    # executables first: captured CUDA graphs hold NCCL work and symmetric-memory buffers that must be released
    # (and the device drained) before the process group is torn down
    for c in _executable_caches:
        for entry in list(c.values()):
            ex = entry[0]
            for attr in ("_graph", "_graph_io"):
                if hasattr(ex, attr):
                    setattr(ex, attr, None)
    clear_executable_cache()
    import gc
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    dm.shutdown_global_cluster()
    is_initialized = False


# ------------------------------------------------------------------------------------------------
# parallelize
# ------------------------------------------------------------------------------------------------
_DYN = object()  # marks a dynamic (tensor) leaf in the flattened argument structure
_TENSOR_LEAF = (torch.Tensor, DistributedArray, ReplicatedDistributedArray, np.ndarray)


def _is_tensor_leaf(x) -> bool:
    return isinstance(x, _TENSOR_LEAF)


def _aval(x):
    if isinstance(x, (DistributedArray, ReplicatedDistributedArray)):
        return (tuple(x.shape), x.dtype, None)
    if isinstance(x, np.ndarray):
        t = torch.from_numpy(x) if x.dtype != np.float64 else torch.from_numpy(x)
        return (tuple(t.shape), t.dtype, None)
    return (tuple(x.shape), x.dtype, None)


_executable_caches = []


def set_seed(seed: int):
    """Seed compile-time and run-time randomness identically on every rank (reference: alpa.set_seed,
    device_mesh.py set_seed :2328-2340 -- the runtime seed feeds the stateful RNG of every mesh worker)."""
    global_config.compile_random_seed = int(seed)
    global_config.runtime_random_seed = int(seed)
    torch.manual_seed(int(seed))
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(int(seed))


def clear_executable_cache():
    """Drop every compiled executable (reference: api.py:236-238)."""
    for c in _executable_caches:
        c.clear()


class ParallelizedFunc:
    """The callable returned by `parallelize` (reference: api.py:106-233)."""

    def __init__(self, fun: Callable, static_argnums, donate_argnums, batch_argnums, method):
        self.fun = fun
        self.static_argnums = static_argnums
        self.donate_argnums = donate_argnums
        self.batch_argnums = batch_argnums
        self.method = method
        self._cache = {}
        self.last_executable = None
        _executable_caches.append(self._cache)
        functools.update_wrapper(self, fun)

    # ---- public
    def __call__(self, *args):
        executable, flat_args, out_tree_cell = self._decode_args_and_get_executable(*args)
        out_flat = executable.launch_on_driver(*flat_args)
        return pytree.tree_unflatten(list(out_flat), out_tree_cell[0])

    def get_executable(self, *args):
        executable, _, _ = self._decode_args_and_get_executable(*args)
        return executable

    def preshard_dynamic_args(self, *args):
        """Shard the dynamic arguments the way the executable wants them (reference: api.py:133-143)."""
        executable, flat_args, _ = self._decode_args_and_get_executable(*args)
        sharded = executable.preshard_dynamic_args(*flat_args)
        return self._rebuild_args(args, sharded)

    def get_last_executable(self):
        return self.last_executable

    # ---- internals
    def _static_set(self, nargs):
        if self.static_argnums == "auto" or self.static_argnums is None:
            return set()
        s = self.static_argnums
        return set([s] if isinstance(s, int) else s)

    def _donate_set(self, args):
        if self.donate_argnums == "auto":
            # the train state (arg 0) is donated when it looks like a TrainState (reference: util.py:70-101)
            from alpa_b200.model.model_util import TrainState
            return {i for i, a in enumerate(args) if isinstance(a, TrainState)}
        if self.donate_argnums is None:
            return set()
        d = self.donate_argnums
        return set([d] if isinstance(d, int) else d)

    def _batch_set(self):
        b = self.batch_argnums
        if b is None:
            return set()
        return set([b] if isinstance(b, int) else b)

    def _rebuild_args(self, args, new_dynamic_leaves):
        it = iter(new_dynamic_leaves)
        out = []
        static = self._static_set(len(args))
        for i, a in enumerate(args):
            if i in static:
                out.append(a)
                continue
            leaves, tree = pytree.tree_flatten(a)
            leaves = [next(it) if _is_tensor_leaf(l) else l for l in leaves]
            out.append(pytree.tree_unflatten(leaves, tree))
        return tuple(out)

    def _decode_args_and_get_executable(self, *args):
        static = self._static_set(len(args))
        donate = self._donate_set(args)
        batch = self._batch_set()
        dyn_leaves, donated, batched = [], [], []
        structure = []  # per arg: ("static", value) | ("dyn", tree, leaf kinds/static leaves)
        key_parts = []
        for i, a in enumerate(args):
            if i in static:
                structure.append(("static", a))
                key_parts.append(("s", _hashable(a)))
                continue
            leaves, tree = pytree.tree_flatten(a)
            kinds = []
            for l in leaves:
                if _is_tensor_leaf(l):
                    kinds.append(_DYN)
                    dyn_leaves.append(l)
                    donated.append(i in donate)
                    batched.append(i in batch)
                else:
                    kinds.append(l)
            structure.append(("dyn", tree, kinds))
            key_parts.append(("d", str(tree), tuple(_hashable(k) for k in kinds if k is not _DYN)))
        avals = tuple(_aval(l) for l in dyn_leaves)
        key = (tuple(key_parts), avals, tuple(donated), tuple(batched), id(self.method))
        entry = self._cache.get(key)
        if entry is None:
            out_tree_cell = [None]

            def flat_fun(*flat):
                it = iter(flat)
                call_args = []
                for st in structure:
                    if st[0] == "static":
                        call_args.append(st[1])
                    else:
                        _, tree, kinds = st
                        leaves = [next(it) if k is _DYN else k for k in kinds]
                        call_args.append(pytree.tree_unflatten(leaves, tree))
                out = self.fun(*call_args)
                out_leaves, out_tree = pytree.tree_flatten(out)
                out_tree_cell[0] = out_tree
                return out_leaves

            # pytree context for methods that need it (manual sharding specs, follow/create-state)
            flat_fun.in_structure = structure
            flat_fun.out_tree_cell = out_tree_cell
            flat_fun.dynamic_leaves = dyn_leaves
            executable = self.method.compile_executable(flat_fun, avals, donated, batched,
                                                        name=getattr(self.fun, "__name__", "fn"))
            entry = (executable, out_tree_cell)
            self._cache[key] = entry
        self.last_executable = entry[0]
        return entry[0], dyn_leaves, entry[1]


def _hashable(x):
    try:
        hash(x)
        return x
    except TypeError:
        return id(x)


def parallelize(fun: Optional[Callable] = None, *, static_argnums: Union[Sequence[int], str] = "auto",
                donate_argnums: Union[Sequence[int], str] = "auto",
                batch_argnums: Union[Sequence[int], str] = (1,), method=None):
    """Parallelise a PyTorch step function (reference: alpa.parallelize, api.py:71-103).

    batch_argnums: positional args whose leading dim is the batch (split across data-parallel devices
    and into micro-batches).  donate_argnums: args whose buffers may be reused for outputs ("auto" =
    the TrainState).  method: a `ParallelMethod` (default ShardParallel())."""

    def decorate(f):
        from alpa_b200.parallel_method import ShardParallel
        m = method if method is not None else ShardParallel()
        return ParallelizedFunc(f, static_argnums, donate_argnums, batch_argnums, m)

    if fun is None:
        return decorate
    return decorate(fun)


# ------------------------------------------------------------------------------------------------
# grad / value_and_grad
# ------------------------------------------------------------------------------------------------
def value_and_grad(fun: Callable, argnums: Union[int, Sequence[int]] = 0, has_aux: bool = False):
    """Like jax.value_and_grad for torch pytrees, traceable (reference: alpa.value_and_grad, api.py:265-287).

    The gradient pytree passes through a `grad` marker so the compiler can split compute-grad from
    apply-grad for gradient accumulation and pipelining (reference: mark_gradient, primitive_def.py:24)."""
    single = isinstance(argnums, int)
    nums = (argnums,) if single else tuple(argnums)

    def wrapped(*args, **kwargs):
        from alpa_b200.parallel.pipeline.primitive_def import (apply_grad_func_transforms, mark_gradient,
                                                                mark_loss)
        f = apply_grad_func_transforms(fun)
        args = list(args)
        trees, all_leaves, leaf_is_tensor = [], [], []
        for n in nums:
            leaves, tree = pytree.tree_flatten(args[n])
            new = []
            for l in leaves:
                if isinstance(l, torch.Tensor) and l.is_floating_point():
                    l = l.detach().requires_grad_(True)
                    all_leaves.append(l)
                new.append(l)
            args[n] = pytree.tree_unflatten(new, tree)
            trees.append((tree, new))
        with torch.enable_grad():
            out = f(*args, **kwargs)
            loss, aux = (out if has_aux else (out, None))
            loss = mark_loss(loss)  # separates the forward from the backward part of the traced graph
            grads = torch.autograd.grad(loss, all_leaves, allow_unused=True)
        grads = [g if g is not None else torch.zeros_like(l) for g, l in zip(grads, all_leaves)]
        grads = mark_gradient(grads)
        it = iter(grads)
        grad_trees = []
        for tree, leaves in trees:
            gl = [next(it) if (isinstance(l, torch.Tensor) and l.is_floating_point()) else None for l in leaves]
            grad_trees.append(pytree.tree_unflatten(gl, tree))
        g = grad_trees[0] if single else tuple(grad_trees)
        loss = loss.detach()
        if has_aux:
            aux = pytree.tree_map(lambda t: t.detach() if isinstance(t, torch.Tensor) else t, aux)
            return (loss, aux), g
        return loss, g

    return wrapped


def grad(fun: Callable, argnums: Union[int, Sequence[int]] = 0, has_aux: bool = False):
    """Gradient of `fun` w.r.t. `argnums` (reference: alpa.grad, api.py:241-262)."""
    vg = value_and_grad(fun, argnums, has_aux)

    def wrapped(*args, **kwargs):
        out, g = vg(*args, **kwargs)
        if has_aux:
            return g, out[1]
        return g

    return wrapped
