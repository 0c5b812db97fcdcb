"""Global configuration (one mutable object, like the reference's alpa/global_env.py:5-139).

Differences that follow from the H100-native design: there is no XLA/Ray, so the XLA memory and
port knobs are replaced by torch.distributed / CUDA-graph / symmetric-memory knobs; every option the
reference exposes for the planner and the pipeline runtime keeps its name.
"""
import os


def _env_flag(name, default=False):
    v = os.environ.get(name)
    if v is None:
        return default
    return v.lower() in ("1", "true", "yes", "on")


class GlobalConfig:
    """Process-wide options.  Every rank holds an identical copy (SPMD, one process per GPU)."""

    def __init__(self):
        # ---------------- device mesh / backend ----------------
        self.backend = "gpu"                      # "gpu" (nccl) or "cpu" (gloo)
        self.compile_random_seed = 42
        self.runtime_random_seed = 42
        self.delete_remote_arrays_threshold = 50
        # Compute dtype policy of the kernel library: bf16 tensors run the sm_90a kernels,
        # everything else (CPU, fp32) runs the PyTorch reference implementation of the same op.
        self.use_native_kernels = True
        # Capture each compiled SPMD program in a CUDA graph after warm-up.
        self.use_cuda_graph = _env_flag("ALPA_B200_CUDA_GRAPH", False)
        # Use NVLink peer-memory fused compute+collective kernels where the plan allows.
        self.use_fused_collectives = _env_flag("ALPA_B200_FUSED_COLLECTIVES", True)
        # tensor parallelism: row-parallel linear + all-reduce as "GEMM into symmetric memory + NVLS reduce"
        # (built from validated kernels; the combined instruction has not run on hardware yet -> opt-in)
        # (reference: global_config.has_cuda -- whether this process sees a CUDA device)
        try:
            import torch as _torch
            self.has_cuda = bool(_torch.cuda.is_available())
        except Exception:  # noqa: BLE001
            self.has_cuda = False
        self.use_fused_linear_allreduce = _env_flag("ALPA_B200_FUSED_LINEAR_ALLREDUCE", False)
        # all-gather (activation rows) + column-parallel linear served by the push + gated-TMA GEMM kernel pair; the
        # lowering rule is always on (on the emulated mesh and by default on GPUs the instruction runs as all-gather +
        # GEMM), the fused kernel call site is opt-in until it has run on hardware
        self.use_fused_allgather_linear = _env_flag("ALPA_B200_FUSED_ALLGATHER_LINEAR", False)
        # GEMM -> reduce-scatter through the peer-store epilogue (ZeRO-2 gradient path): wins at 2 GPUs (20.4 vs 21.2 ms),
        # loses at 8 (25.7 vs 21.9 ms) and allocates one symmetric workspace per call site -> opt-in; the instruction
        # otherwise runs as GEMM + NCCL reduce-scatter
        self.use_fused_linear_reduce_scatter = _env_flag("ALPA_B200_FUSED_LINEAR_REDUCE_SCATTER", False)
        # data-parallel gradient sync through NVSwitch in-network reduction (multimem) instead of NCCL
        self.use_nvls_grad_allreduce = _env_flag("ALPA_B200_NVLS_GRAD_ALLREDUCE", False)
        # pack gradients into 128 MiB buckets: one NCCL all-reduce per bucket instead of one per parameter
        self.use_bucketed_grad_allreduce = _env_flag("ALPA_B200_BUCKETED_GRAD_ALLREDUCE", False)
        # static gradient buckets: every data-parallel gradient lives in a slice of a persistent flat buffer and ONE
        # all-reduce per bucket is launched as soon as its last member exists (graph-capturable, no pack/unpack)
        self.use_static_grad_buckets = _env_flag("ALPA_B200_STATIC_GRAD_BUCKETS", True)
        self.grad_bucket_bytes = int(os.environ.get("ALPA_B200_GRAD_BUCKET_BYTES", str(128 << 20)))
        # a full gradient bucket is reduced under the next kernel whose name contains one of these (compute-bound
        # kernels: the reduction's memory traffic does not slow them), at the latest `grad_reduce_max_hold` instructions on
        self.grad_reduce_overlap_ops = ("attention",)
        self.grad_reduce_max_hold = 64
        # sharded (ZeRO-3) parameters: issue their all-gather this many instructions ahead of the consumer
        self.param_allgather_prefetch_distance = 24

        # ---------------- shard parallel ----------------
        self.shard_parallel_sync_for_timer = False

        # ---------------- pipeline parallel (compile) ----------------
        self.debug_with_pipeshard_runtime = False
        self.profile_with_whole_ray_cluster = True   # kept for API parity; unused (no Ray)
        self.profile_timeout = 500
        self.profile_maximum_retry = 2
        self.overwrite_submesh_choices = None
        self.always_donate_micro_batch_vars = True

        # ---------------- pipeline runtime ----------------
        self.pipeline_sync_for_timer = False
        self.pipeline_distributed_compile = True
        self.eagerly_create_communicators = True
        self.pipeline_check_alive = False
        self.pipeline_use_signal_send_recv = False
        # cross-mesh transfers on dedicated send / receive streams, ordered by per-value done / ready events
        self.pipeline_async_comm = _env_flag("ALPA_B200_PIPELINE_ASYNC_COMM", True)
        # cross-mesh transfers through the native communication groups (csrc/comm_group.cpp: per-pair NCCL communicators
        # with per-direction streams, uuid events) instead of torch.distributed p2p.  Opt-in: not yet run on hardware.
        self.use_native_comm_group = _env_flag("ALPA_B200_NATIVE_COMM", False)
        self.native_comm_backend = None               # test hook: an object with the `_planner.comm` interface
        self.use_local_allgather = True
        self.resharding_mode = "send_recv"            # or "broadcast"
        self.nccl_mode = "torch"                      # torch.distributed ProcessGroupNCCL
        self.enable_overlapping = False
        self.resharding_loadbalance_mode = "normal"   # normal|no_loadbalance|loadbalance_size|loadbalance_order
        self.loadbalance_order_algo = "greedy"

        # ---------------- benchmark ----------------
        self.use_dummy_value_for_benchmarking = False

        # ---------------- logging ----------------
        self.print_compilation_time = False
        self.print_auto_layer_stats = False
        self.collect_trace = False

    def update_worker_config(self, cfg: "GlobalConfig"):
        """Copy the runtime-relevant fields of `cfg` (reference: global_env.py:108-136)."""
        for k in ("backend", "compile_random_seed", "runtime_random_seed", "pipeline_sync_for_timer",
                  "pipeline_use_signal_send_recv", "use_local_allgather", "resharding_mode",
                  "nccl_mode", "enable_overlapping", "collect_trace", "use_cuda_graph",
                  "use_fused_collectives"):
            setattr(self, k, getattr(cfg, k))


global_config = GlobalConfig()

# True inside worker-only helper processes (kept for API parity with alpa.global_env.is_worker).
is_worker = _env_flag("ALPA_IS_WORKER", False)
