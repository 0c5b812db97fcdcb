"""Cluster profiling database and the analytic cost model that feeds the planners.

Reference: alpa/mesh_profiling.py (MeshProfilingResult:18, ProfilingResultDatabase:162, profile_one_hlo_op:392,
enumerate_all_collective_spec:668, profile_all:725, estimate_hlo_module_cost:901) and the C++ HLO cost model
(XLA/service/gpu/gpu_cost_model.cc).  The reference micro-benchmarks XLA executables (dot, all-reduce,
all-gather, reduce-scatter, all-to-all) and interpolates; here the same tables are filled by timing *our*
kernels and NCCL collectives with CUDA events; without them the H100 data-sheet defaults of `CostModel` apply,
overridden by a measured MEASURED_PEAKS.json when one is present.
"""
from __future__ import annotations

import json
import os
import pickle
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

import logging
logger = logging.getLogger(__name__)


class MeshProfilingResult:
    """Cost tables of one mesh shape: op -> [(size key, seconds)]."""

    def __init__(self):
        self.dot_cost_dict: Dict[Tuple, List[Tuple[float, float]]] = {}
        self.all_reduce_cost_dict: Dict[Tuple, List[Tuple[float, float]]] = {}
        self.all_gather_cost_dict: Dict[Tuple, List[Tuple[float, float]]] = {}
        self.reduce_scatter_cost_dict: Dict[Tuple, List[Tuple[float, float]]] = {}
        self.all_to_all_cost_dict: Dict[Tuple, List[Tuple[float, float]]] = {}
        self.available_memory_per_device: Optional[float] = None
        # (op, group size, dtype, bytes) of measurements that raised on every attempt: persisted with the database
        # so a re-run does not walk into the same failure again (reference: mesh_profiling.py:803-844)
        self.failed_keys: set = set()

    def update(self, other: "MeshProfilingResult"):
        for name in ("dot", "all_reduce", "all_gather", "reduce_scatter", "all_to_all"):
            getattr(self, f"{name}_cost_dict").update(getattr(other, f"{name}_cost_dict"))
        if other.available_memory_per_device is not None:
            self.available_memory_per_device = other.available_memory_per_device
        self.failed_keys |= getattr(other, "failed_keys", set())

    def sort_cost_lists(self):
        """Sort every cost table by size (reference: MeshProfilingResult.sort_cost_lists)."""
        for name in ("dot", "all_reduce", "all_gather", "reduce_scatter", "all_to_all"):
            d = getattr(self, f"{name}_cost_dict")
            for k in d:
                d[k] = sorted(d[k])

    def make_monotonic(self):
        """Measured tables can dip (noise, protocol switches): make the cost non-decreasing in the size so that the
        interpolated model never prefers a larger message (reference: MeshProfilingResult.make_monotonic)."""
        self.sort_cost_lists()
        for name in ("dot", "all_reduce", "all_gather", "reduce_scatter", "all_to_all"):
            d = getattr(self, f"{name}_cost_dict")
            for k, tab in d.items():
                out, hi = [], 0.0
                for size, t in tab:
                    hi = max(hi, t)
                    out.append((size, hi))
                d[k] = out

    def __setstate__(self, state):          # databases pickled before `failed_keys` existed
        self.__dict__.update(state)
        self.__dict__.setdefault("failed_keys", set())

    @staticmethod
    def _interp(table: List[Tuple[float, float]], size: float) -> float:
        if not table:
            return 0.0
        xs = np.array([t[0] for t in table], dtype=np.float64)
        ys = np.array([t[1] for t in table], dtype=np.float64)
        order = np.argsort(xs)
        xs, ys = xs[order], ys[order]
        if size <= xs[0]:
            return float(ys[0])
        if size >= xs[-1]:
            return float(ys[-1] * size / xs[-1])
        return float(np.interp(size, xs, ys))

    def estimate_all_reduce(self, group_size: int, dtype: str, num_bytes: float) -> float:
        return self._interp(self.all_reduce_cost_dict.get((group_size, dtype), []), num_bytes)

    def estimate_all_gather(self, group_size: int, dtype: str, num_bytes: float) -> float:
        return self._interp(self.all_gather_cost_dict.get((group_size, dtype), []), num_bytes)

    def estimate_reduce_scatter(self, group_size: int, dtype: str, num_bytes: float) -> float:
        return self._interp(self.reduce_scatter_cost_dict.get((group_size, dtype), []), num_bytes)

    def estimate_all_to_all(self, group_size: int, dtype: str, num_bytes: float) -> float:
        return self._interp(self.all_to_all_cost_dict.get((group_size, dtype), []), num_bytes)

    def estimate_dot(self, dtype: str, flops: float) -> float:
        return self._interp(self.dot_cost_dict.get((dtype,), []), flops)

    def __str__(self):
        return (f"MeshProfilingResult(dot={len(self.dot_cost_dict)}, ar={len(self.all_reduce_cost_dict)}, "
                f"ag={len(self.all_gather_cost_dict)}, rs={len(self.reduce_scatter_cost_dict)}, "
                f"a2a={len(self.all_to_all_cost_dict)})")


class ProfilingResultDatabase:
    """(cluster key, mesh shape) -> MeshProfilingResult, picklable (reference: mesh_profiling.py:162-206)."""

    def __init__(self, data: Optional[dict] = None):
        self.data: Dict[Tuple[str, Tuple[int, int]], MeshProfilingResult] = data or {}

    def query(self, cluster_key: str, mesh_shape: Tuple[int, int]) -> Optional[MeshProfilingResult]:
        return self.data.get((cluster_key, tuple(mesh_shape)))

    def update_one_mesh(self, cluster_key: str, mesh_shape, result: MeshProfilingResult):
        key = (cluster_key, tuple(mesh_shape))
        if key in self.data:
            self.data[key].update(result)
        else:
            self.data[key] = result

    def update(self, other: "ProfilingResultDatabase"):
        for (k, s), v in other.data.items():
            self.update_one_mesh(k, s, v)

    def insert_dummy_mesh_result(self, cluster_key: str, mesh_shape):
        """A result filled from the analytic model, for meshes that could not be profiled (reference:
        ProfilingResultDatabase.insert_dummy_mesh_result)."""
        cm = default_cost_model()
        n = int(mesh_shape[0]) * int(mesh_shape[1])
        res = MeshProfilingResult()
        sizes = [float(1 << lg) for lg in range(10, 31, 2)]
        res.dot_cost_dict[("bf16",)] = [(2.0 * d ** 3, cm.gemm_seconds(2.0 * d ** 3)) for d in (1024, 2048, 4096, 8192)]
        if n > 1:
            res.all_reduce_cost_dict[(n, "bf16")] = [(s_, cm.all_reduce_seconds(s_, n)) for s_ in sizes]
            res.all_gather_cost_dict[(n, "bf16")] = [(s_, cm.all_gather_seconds(s_, n)) for s_ in sizes]
            res.reduce_scatter_cost_dict[(n, "bf16")] = [(s_, cm.all_gather_seconds(s_, n)) for s_ in sizes]
            res.all_to_all_cost_dict[(n, "bf16")] = [(s_, cm.all_to_all_seconds(s_, n)) for s_ in sizes]
        self.update_one_mesh(cluster_key, tuple(mesh_shape), res)
        return res

    def save(self, filename: str):
        with open(filename, "wb") as f:
            pickle.dump(self.data, f)

    def load(self, filename: str):
        with open(filename, "rb") as f:
            self.update(ProfilingResultDatabase(pickle.load(f)))

    def __str__(self):
        return "\n".join(f"{k}: {v}" for k, v in self.data.items())


# ------------------------------------------------------------------------------------------------
# analytic model.  Defaults are NVIDIA data-sheet figures of the H100 SXM (80 GB HBM3, 700 W), not measurements:
# peak rates are upper bounds, so a measured MEASURED_PEAKS.json (or a profiled database) replaces them when present.
# ------------------------------------------------------------------------------------------------
@dataclass
class CostModel:
    flops_per_second: float = 989e12          # dense bf16 tensor-core peak (data sheet)
    hbm_bytes_per_second: float = 3.35e12     # HBM3 (data sheet)
    nvlink_bytes_per_second: float = 4.5e11   # NVLink 4: 900 GB/s bidirectional = 450 GB/s per direction per GPU
    allreduce_bus_bytes_per_second: float = 4.5e11   # bus bandwidth bound by the per-direction link rate
    collective_latency: float = 12e-6         # assumed per-collective launch + synchronisation latency
    memory_bytes: float = 80e9                # HBM capacity per GPU

    def all_reduce_seconds(self, num_bytes: float, n: int) -> float:
        if n <= 1:
            return 0.0
        return self.collective_latency + 2 * (n - 1) / n * num_bytes / self.allreduce_bus_bytes_per_second

    def all_gather_seconds(self, num_bytes: float, n: int) -> float:
        if n <= 1:
            return 0.0
        return self.collective_latency + (n - 1) / n * num_bytes / self.nvlink_bytes_per_second

    reduce_scatter_seconds = all_gather_seconds

    def all_to_all_seconds(self, num_bytes: float, n: int) -> float:
        if n <= 1:
            return 0.0
        return self.collective_latency + (n - 1) / n * num_bytes / n / self.nvlink_bytes_per_second * 1.0

    def p2p_seconds(self, num_bytes: float) -> float:
        return self.collective_latency + num_bytes / self.nvlink_bytes_per_second

    def gemm_seconds(self, flops: float) -> float:
        return flops / self.flops_per_second

    def to_alpha_beta(self):
        """(alpha, beta) of the planner's LogicalDeviceMesh cost formulas: seconds and seconds/byte."""
        return self.collective_latency, 1.0 / self.nvlink_bytes_per_second


def native_cost_tables(cm: Optional["CostModel"] = None, prof: Optional["MeshProfilingResult"] = None):
    """`alpa_b200._planner.CostTables` (C++ cost model, csrc/cost_model.cpp) filled from the peak-rate model and, when
    given, from the profiled collective tables (reference: the profiling DB feeds gpu_cost_model.cc)."""
    from alpa_b200.parallel.shard.auto_sharding import planner_module
    P = planner_module()
    cm = cm or default_cost_model()
    t = P.CostTables()
    t.flops_per_second = cm.flops_per_second
    t.hbm_bytes_per_second = cm.hbm_bytes_per_second
    t.link_bytes_per_second = cm.nvlink_bytes_per_second
    t.allreduce_bus_bytes_per_second = cm.allreduce_bus_bytes_per_second
    t.latency = cm.collective_latency
    if prof is not None:
        for kind, d in ((P.K_ALL_REDUCE, prof.all_reduce_cost_dict), (P.K_ALL_GATHER, prof.all_gather_cost_dict),
                        (P.K_REDUCE_SCATTER, prof.reduce_scatter_cost_dict), (P.K_ALL_TO_ALL, prof.all_to_all_cost_dict)):
            for (n, _dtype), table in d.items():
                for (size, sec) in table:
                    t.add(kind, int(n), float(size), float(sec))
        for (_key), table in getattr(prof, "dot_cost_dict", {}).items():
            for (size, sec) in table:
                t.add(P.K_DOT, 1, float(size), float(sec))
    return t


_default_cm: Optional[CostModel] = None


def default_cost_model() -> CostModel:
    global _default_cm
    if _default_cm is None:
        cm = CostModel()
        path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
        try:
            with open(path) as f:
                p = json.load(f)
            cm.flops_per_second = float(p.get("bf16_tflops_sustained", cm.flops_per_second / 1e12)) * 1e12
            cm.hbm_bytes_per_second = float(p.get("hbm_gbs", cm.hbm_bytes_per_second / 1e9)) * 1e9
        except Exception:  # noqa: BLE001
            pass
        _default_cm = cm
    return _default_cm


def set_cost_model(cm: CostModel):
    global _default_cm
    _default_cm = cm


# ------------------------------------------------------------------------------------------------
# on-device profiling (run inside a torchrun job on the GPU node)
# ------------------------------------------------------------------------------------------------
def _time_cuda(fn, warmup=3, iters=10) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters / 1e3


def _time_host(fn, warmup=1, iters=3) -> float:
    """Wall-clock timing for the CPU (gloo) backend -- only used to exercise the profiling flow without GPUs."""
    import time
    for _ in range(warmup):
        fn()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    return (time.perf_counter() - t0) / iters


_DTYPES = {"bf16": torch.bfloat16, "f32": torch.float32}


def enumerate_collective_specs(group_size: int, max_comm_size_log2: int, min_comm_size_log2: int = 10, step: int = 2,
                               dtypes: Sequence[str] = ("bf16", "f32")):
    """Every (op, group size, dtype, bytes) a mesh profile measures (reference: enumerate_all_collective_spec,
    mesh_profiling.py:668-722)."""
    specs = []
    for op in ("all_reduce", "all_gather", "reduce_scatter", "all_to_all"):
        for dt in dtypes:
            for lg in range(min_comm_size_log2, max_comm_size_log2 + 1, step):
                specs.append((op, group_size, dt, 1 << lg))
    return specs


def profile_one_mesh(group_ranks: Sequence[int], max_comm_size_log2: int = 28, dot_sizes=(1024, 2048, 4096, 8192),
                     skip_keys: Optional[set] = None, max_retry: int = 2, min_comm_size_log2: int = 10,
                     dtypes: Sequence[str] = ("bf16", "f32")) -> MeshProfilingResult:
    """Time bf16 GEMMs (our wgmma kernel) and the collectives of `enumerate_collective_specs` over `group_ranks`
    (reference: profile_one_hlo_op / profile_hlo_ops, mesh_profiling.py:392-665).  Every measurement is retried up to
    `max_retry` times; one that keeps failing (out of memory at the largest sizes, an unsupported dtype on a backend)
    is recorded in `failed_keys` and skipped -- the profile of the mesh still completes.  Keys in `skip_keys` (failures
    remembered from an earlier run) are not attempted.  The group agrees on success / failure of each measurement, so
    no rank is left alone inside a collective."""
    import torch.distributed as dist
    res = MeshProfilingResult()
    cuda = torch.cuda.is_available() and (not dist.is_initialized() or dist.get_backend() == "nccl")
    dev = torch.device("cuda", torch.cuda.current_device()) if cuda else torch.device("cpu")
    timer = _time_cuda if cuda else _time_host
    skip_keys = skip_keys or set()
    fail_inject = set(filter(None, os.environ.get("ALPA_B200_PROFILE_FAIL", "").split(",")))      # tests
    n = len(group_ranks)
    group = None
    if n > 1 and dist.is_initialized():
        from alpa_b200.device_mesh import DistCommunicator
        group = DistCommunicator.get_group(tuple(group_ranks))

    def robust(key, make_fn):
        """Seconds, or None after `max_retry` + 1 failed attempts (agreed on by the whole group)."""
        if key in skip_keys:
            res.failed_keys.add(key)
            return None
        for attempt in range(max_retry + 1):
            ok, t = 1.0, 0.0
            try:
                if key[0] in fail_inject:
                    raise RuntimeError(f"injected failure of {key[0]}")
                t = timer(make_fn())
            except (RuntimeError, ValueError) as e:
                ok = 0.0
                logger.warning("profiling %s failed (attempt %d): %s", key, attempt, e)
                if cuda:
                    torch.cuda.empty_cache()
            if group is not None:
                flag = torch.tensor([ok], device=dev)
                dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)
                ok = float(flag[0])
            if ok > 0:
                return t
        res.failed_keys.add(key)
        return None

    if cuda:
        from alpa_b200 import ops
        C = ops.native_module()
        table = []
        for d in dot_sizes:
            def mk(d=d):
                a = torch.randn(d, d, device=dev, dtype=torch.bfloat16)
                b = torch.randn(d, d, device=dev, dtype=torch.bfloat16)
                return lambda: C.gemm(a, b, False, False)
            t = robust(("dot", 1, "bf16", d), mk)
            if t is not None:
                table.append((2.0 * d ** 3, t))
        res.dot_cost_dict[("bf16",)] = table
        free, _ = torch.cuda.mem_get_info()
        res.available_memory_per_device = float(free)
    if group is not None:
        tables: Dict[Tuple[str, str], List[Tuple[float, float]]] = {}
        for key in enumerate_collective_specs(n, max_comm_size_log2, min_comm_size_log2, 2, dtypes):
            op, _, dt, nbytes = key
            dtype = _DTYPES[dt]
            numel = nbytes // torch.empty((), dtype=dtype).element_size()

            def mk(op=op, dtype=dtype, numel=numel):
                x = torch.zeros(numel, device=dev, dtype=dtype)
                if op == "all_reduce":
                    return lambda: dist.all_reduce(x, group=group)
                out = torch.zeros(n * numel, device=dev, dtype=dtype)
                if op == "all_gather":
                    return lambda: dist.all_gather_into_tensor(out, x, group=group)
                if op == "reduce_scatter":
                    return lambda: dist.reduce_scatter_tensor(x, out, group=group)
                y = torch.zeros_like(out)
                return lambda: dist.all_to_all_single(y, out, group=group)
            t = robust(key, mk)
            if t is not None:
                tables.setdefault((op, dt), []).append((nbytes if op == "all_reduce" else nbytes * n, t))
        for (op, dt), tab in tables.items():
            getattr(res, f"{op}_cost_dict")[(n, dt)] = tab
    return res


def profile_all(device_cluster, cluster_key: str = "b200", max_comm_size_intra_node: int = 28,
                max_comm_size_inter_node: int = 26, cache_filename: Optional[str] = None, retry_failed: bool = False,
                **kwargs) -> ProfilingResultDatabase:
    """Profile every power-of-two submesh of the cluster (reference: profile_all, mesh_profiling.py:725-898).

    Resumable: meshes already in `cache_filename` are not profiled again, the cache is rewritten after every mesh, and
    measurements that failed before are skipped unless `retry_failed`."""
    import torch.distributed as dist
    db = ProfilingResultDatabase()
    if cache_filename and os.path.exists(cache_filename):
        db.load(cache_filename)
    n = device_cluster.num_devices_per_host
    rank = dist.get_rank() if dist.is_initialized() else 0
    size = 1
    while size <= n:
        base = (rank // size) * size
        ranks = list(range(base, base + size))
        # every rank participates in the group of its own block; blocks run concurrently like the
        # reference's submesh profiling
        if dist.is_initialized() and size > 1:
            from alpa_b200.device_mesh import DistCommunicator
            for b in range(0, dist.get_world_size(), size):
                DistCommunicator.get_group(tuple(range(b, b + size)))
        old = db.query(cluster_key, (1, size))
        done = old is not None and (old.all_reduce_cost_dict or size == 1) and not (retry_failed and old.failed_keys)
        if not done:
            skip = set() if (retry_failed or old is None) else set(old.failed_keys)
            res = profile_one_mesh(ranks, max_comm_size_intra_node, skip_keys=skip, **kwargs)
            if old is not None and retry_failed:
                old.failed_keys = set()
            db.update_one_mesh(cluster_key, (1, size), res)
            if cache_filename and rank == 0:
                db.save(cache_filename)                      # after every mesh: an interrupted run resumes here
        size *= 2
    return db


def estimate_stage_cost_from_db(db: ProfilingResultDatabase, cluster_key: str, mesh_shape, flops: float,
                                collectives: Sequence[Tuple[str, int, float]]) -> float:
    """Latency of a stage = GEMM FLOPs at the profiled rate + its collectives by table interpolation
    (reference: estimate_hlo_module_cost, mesh_profiling.py:901-913 / gpu_cost_model.cc:258-341)."""
    res = db.query(cluster_key, mesh_shape)
    cm = default_cost_model()
    if res is None:
        t = cm.gemm_seconds(flops)
        for kind, n, nbytes in collectives:
            t += getattr(cm, f"{kind}_seconds")(nbytes, n)
        return t
    t = res.estimate_dot("bf16", flops) or cm.gemm_seconds(flops)
    for kind, n, nbytes in collectives:
        est = getattr(res, f"estimate_{kind}")(n, "bf16", nbytes)
        t += est if est > 0 else getattr(cm, f"{kind}_seconds")(nbytes, n)
    return t


# names of the reference's module (alpa/mesh_profiling.py)
enumerate_all_collective_spec = enumerate_collective_specs
estimate_hlo_module_cost = estimate_stage_cost_from_db


def profile_dot(sizes=(1024, 2048, 4096, 8192)):
    """[(flops, seconds)] of square bf16 GEMMs with this package's wgmma kernel (reference: profile_dot)."""
    res = profile_one_mesh([0], max_comm_size_log2=0, dot_sizes=tuple(sizes))
    return res.dot_cost_dict.get(("bf16",), [])
