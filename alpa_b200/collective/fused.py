"""Fused compute + collective operators over NVLink peer memory (symmetric memory).

These are the H100-native replacements for "cuBLAS GEMM then NCCL collective" (the reference's K3/K5:
out-projection / MLP-down GEMM followed by all-reduce or reduce-scatter, and K1/K4: all-gather followed by
the QKV / MLP-up GEMM; XLA/service/gpu/nccl_all_reduce_thunk.cc:103-121,:434-458, nccl_all_gather_thunk.cc).

* ``FusedLinearReduceScatter``: y_shard = reduce_scatter(x_local @ w_local^T).  The GEMM epilogue
  stores every partial tile directly into the owning GPU's staging buffer (peer store over NVLink) and
  bumps an arrival counter; a small reduce kernel on the owner sums the tp slots (+bias, +residual).
* ``FusedAllGatherLinear``: y = all_gather(x_shard) @ w_local^T.  A push kernel on a side stream writes the
  local shard into every peer's gather buffer and publishes per-128-row epoch flags; the GEMM's TMA
  producer waits on the flag of the M block it is about to load and starts with the local rows.
* ``multimem_all_reduce``: in-switch (NVLS) all-reduce of a symmetric buffer.

All buffers are double-buffered; counters/epochs are cumulative so no reset traffic is needed.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist


def _symm():
    import torch.distributed._symmetric_memory as symm_mem
    return symm_mem


class SymmWorkspace:
    """A byte buffer mapped into every rank of `group` (CUDA VMM / IPC via torch symmetric memory)."""

    def __init__(self, group, nbytes: int):
        sm = _symm()
        self.group = group
        self.device = torch.device("cuda", torch.cuda.current_device())
        self.nbytes = int((nbytes + 1023) // 1024 * 1024)
        self.buf = sm.empty(self.nbytes, dtype=torch.uint8, device=self.device)
        self.buf.zero_()
        self.hdl = sm.rendezvous(self.buf, group=group)
        self.rank = self.hdl.rank
        self.world = self.hdl.world_size
        self.ptrs: List[int] = [int(p) for p in self.hdl.buffer_ptrs]
        self.multicast_ptr = int(getattr(self.hdl, "multicast_ptr", 0) or 0)
        torch.cuda.synchronize()
        self.hdl.barrier()

    def local(self, offset: int, shape, dtype) -> torch.Tensor:
        n = 1
        for s in shape:
            n *= s
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        return self.buf[offset:offset + nbytes].view(dtype).view(*shape)

    def peer_ptrs(self, offset: int) -> List[int]:
        return [p + offset for p in self.ptrs]

    def barrier(self):
        self.hdl.barrier()


_workspaces: Dict[Tuple, object] = {}


class FusedLinearReduceScatter:
    """y[M/tp, N] (this rank's rows) = sum over ranks of (x_r[M, K_r] @ w_r[N, K_r]^T)."""

    def __init__(self, group, M: int, N: int):
        from alpa_b200 import ops
        self.C = ops.native_module()
        self.tp = dist.get_world_size(group)
        assert M % self.tp == 0 and (M // self.tp) % 32 == 0 and N % 8 == 0, (M, N, self.tp)
        self.M, self.N = M, N
        self.rows = M // self.tp
        self.nblocks32 = self.rows // 32
        self.stage_bytes = self.tp * self.rows * N * 2
        self.flag_bytes = (self.nblocks32 * 4 + 255) // 256 * 256
        self.ws = SymmWorkspace(group, 2 * (self.stage_bytes + self.flag_bytes))
        self.rank = self.ws.rank
        self.calls = 0
        self.cum = [0, 0]
        self.num_n_blocks = (N + 255) // 256
        blocks_per_rank = max(1, self.rows // 128)
        self.rotate = ((self.rank + 1) % self.tp) * blocks_per_rank

    def _offsets(self, b):
        base = b * (self.stage_bytes + self.flag_bytes)
        return base, base + self.stage_bytes

    def __call__(self, x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None,
                 residual: Optional[torch.Tensor] = None, trans_a: bool = False, trans_b: bool = False) -> torch.Tensor:
        """x: [M, K] (or [K, M] with trans_a); w: [N, K] (or [K, N] with trans_b)"""
        b = self.calls & 1
        self.calls += 1
        so, fo = self._offsets(b)
        self.C.gemm_scatter(x, w, trans_b, self.ws.peer_ptrs(so), self.ws.peer_ptrs(fo), self.rank, self.rows, self.N,
                            self.rotate, 0, trans_a)
        self.cum[b] += self.num_n_blocks * self.tp
        out = torch.empty(self.rows, self.N, device=x.device, dtype=torch.bfloat16)
        self.C.rs_reduce(self.ws.ptrs[self.rank] + so, self.ws.ptrs[self.rank] + fo, self.cum[b], out, bias, residual,
                         self.tp, self.rows * self.N)
        return out


class FusedAllGatherLinear:
    """y[tp*Ml, N_local] = all_gather(x_local[Ml, K]) @ w_local[N_local, K]^T (+bias, activation)."""

    def __init__(self, group, M_local: int, K: int):
        from alpa_b200 import ops
        self.C = ops.native_module()
        self.tp = dist.get_world_size(group)
        assert M_local % 128 == 0 and K % 8 == 0, (M_local, K)
        self.Ml, self.K = M_local, K
        self.blocks = M_local // 128
        self.data_bytes = self.tp * M_local * K * 2
        self.flag_bytes = (self.tp * self.blocks * 4 + 255) // 256 * 256
        self.ws = SymmWorkspace(group, 2 * (self.data_bytes + self.flag_bytes))
        self.rank = self.ws.rank
        self.calls = 0
        self.epoch = [0, 0]
        self.push_stream = torch.cuda.Stream()

    def _offsets(self, b):
        base = b * (self.data_bytes + self.flag_bytes)
        return base, base + self.data_bytes

    def __call__(self, x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, act: str = "none",
                 aux_out: Optional[torch.Tensor] = None) -> torch.Tensor:
        b = self.calls & 1
        self.calls += 1
        do, fo = self._offsets(b)
        self.epoch[b] += 1
        ep = self.epoch[b]
        cur = torch.cuda.current_stream()
        ev = torch.cuda.Event()
        ev.record(cur)
        with torch.cuda.stream(self.push_stream):
            self.push_stream.wait_event(ev)
            self.C.ag_push(x, self.ws.peer_ptrs(do), self.ws.peer_ptrs(fo), self.rank, ep, True)
        x.record_stream(self.push_stream)
        gathered = self.ws.local(do, (self.tp * self.Ml, self.K), torch.bfloat16)
        y = self.C.gemm_wait_a(gathered, w, False, self.ws.ptrs[self.rank] + fo, ep, 0, 0,
                               self.rank * self.blocks, bias, aux_out, {"none": 0, "gelu": 1, "relu": 2}[act])
        return y

    def gathered(self, b: Optional[int] = None) -> torch.Tensor:
        b = (self.calls - 1) & 1 if b is None else b
        do, _ = self._offsets(b)
        return self.ws.local(do, (self.tp * self.Ml, self.K), torch.bfloat16)


class MultimemAllReduce:
    """In-place NVLS all-reduce of a bf16 tensor living in symmetric memory."""

    def __init__(self, group, numel: int):
        from alpa_b200 import ops
        self.C = ops.native_module()
        self.ws = SymmWorkspace(group, numel * 2)
        self.numel = numel
        self.tp = self.ws.world
        self.tensor = self.ws.local(0, (numel,), torch.bfloat16)

    @property
    def available(self) -> bool:
        return self.ws.multicast_ptr != 0

    def __call__(self) -> torch.Tensor:
        self.ws.barrier()
        self.C.allreduce_multimem(self.ws.multicast_ptr, self.numel, self.ws.rank, self.tp)
        self.ws.barrier()
        return self.tensor


def get_fused_linear_rs(group, M: int, N: int) -> FusedLinearReduceScatter:
    key = ("rs", id(group), M, N)
    if key not in _workspaces:
        _workspaces[key] = FusedLinearReduceScatter(group, M, N)
    return _workspaces[key]


def get_fused_ag_linear(group, M_local: int, K: int) -> FusedAllGatherLinear:
    key = ("ag", id(group), M_local, K)
    if key not in _workspaces:
        _workspaces[key] = FusedAllGatherLinear(group, M_local, K)
    return _workspaces[key]


# ---------------------------------------------------------------------------------------------------------
# MoE: dispatch / combine kernels that *are* the expert all-to-all (tokens stored into / read from the owning
# GPU's expert buffer over NVLink peer mappings).  One symmetric buffer per call site of the lowered program
# (the program is static, so sites are static): no copies out of symmetric memory, no buffer recycling hazards
# across the forward/backward lifetime of the dispatched tensor.
# ---------------------------------------------------------------------------------------------------------
class FusedMoEDispatch:
    """d_local[E/n, G_total*C, M] <- every rank's routed tokens (x_local: [G_local, S, M])."""

    def __init__(self, group, E: int, G_local: int, C: int, M: int):
        from alpa_b200 import ops
        self.C_ = ops.native_module()
        self.n = dist.get_world_size(group)
        assert E % self.n == 0
        self.E, self.Gl, self.cap, self.M = E, G_local, C, M
        self.shape = (E // self.n, self.n * G_local * C, M)
        self.ws = SymmWorkspace(group, self.shape[0] * self.shape[1] * M * 2)
        self.rank = self.ws.rank
        self.buf = self.ws.local(0, self.shape, torch.bfloat16)

    def __call__(self, x, expert, slot, weight=None) -> torch.Tensor:
        self.buf.zero_()
        self.ws.barrier()          # every peer's buffer is cleared (and no longer read) before anyone stores
        self.C_.moe_dispatch_(x.contiguous(), expert.contiguous(), slot.contiguous(),
                              None if weight is None else weight.contiguous(), self.buf, self.cap,
                              self.ws.peer_ptrs(0), self.rank * self.Gl)
        self.ws.barrier()          # all tokens have landed
        return self.buf


class FusedMoECombine:
    """out[G_local, S, M] = sum_k w_k * eo[peer(e_k)][...] with eo_local: [E/n, G_total*C, M] on every rank."""

    def __init__(self, group, E_local: int, rows: int, M: int):
        from alpa_b200 import ops
        self.C_ = ops.native_module()
        self.n = dist.get_world_size(group)
        self.shape = (E_local, rows, M)
        self.ws = SymmWorkspace(group, E_local * rows * M * 2)
        self.rank = self.ws.rank
        self.buf = self.ws.local(0, self.shape, torch.bfloat16)

    def stage(self, eo: torch.Tensor):
        self.ws.barrier()          # peers finished reading the previous contents
        if eo.data_ptr() != self.buf.data_ptr():
            self.buf.copy_(eo)
        self.ws.barrier()          # every peer's expert output is visible

    def combine(self, eo, expert, slot, weight=None) -> torch.Tensor:
        self.stage(eo)
        G_local = expert.shape[0]
        return self.C_.moe_combine(self.buf, expert.contiguous(), slot.contiguous(),
                                   None if weight is None else weight.contiguous(), self.ws.peer_ptrs(0),
                                   self.rank * G_local)

    def combine_wgrad(self, dout, eo, expert, slot) -> torch.Tensor:
        self.stage(eo)
        G_local = expert.shape[0]
        return self.C_.moe_combine_wgrad(dout.contiguous(), self.buf, expert.contiguous(), slot.contiguous(),
                                         self.ws.peer_ptrs(0), self.rank * G_local)


# ---------------------------------------------------------------------------------------------------------
# Data-parallel gradient all-reduce on the NVSwitch (NVLS): gradients are packed into a symmetric bucket on a side
# stream as backward produces them, reduced *inside the switch* by multimem.ld_reduce / multimem.st with a few CTAs
# (the rest of the GPU keeps computing), and unpacked.  Replaces one NCCL ring/tree all-reduce per gradient
# (reference: XLA all-reduce thunks after backward, K10 of SURVEY.md §2.5).
# ---------------------------------------------------------------------------------------------------------
class _EventWork:
    """Work handle of a collective issued on a side stream: wait() makes the current stream wait for it."""

    def __init__(self, event):
        self.event = event

    def wait(self):
        torch.cuda.current_stream().wait_event(self.event)


class NvlsBucketArena:
    """All bf16 gradient buckets of one lowered program in ONE symmetric-memory allocation (one rendezvous), reduced
    inside the NVSwitch: per bucket `peer_barrier_auto` (every rank's gradients are in place), `allreduce_multimem`
    (each rank reduces 1/n of the slice with multimem.ld_reduce and broadcasts it with multimem.st; a few CTAs, the
    rest of the GPU keeps running backward), `peer_barrier_auto` (every slice has landed).  Barrier epochs live in
    device memory, nothing is allocated or computed on the host per call: the sequence is captured into the step's
    CUDA graph as a side-stream branch.  (replaces: one NCCL ring/tree all-reduce per gradient, reference K10.)"""

    FLAG_BYTES = 1024

    def __init__(self, group, plans, ctas: int = 6, tail_ctas: int = 48):
        # `ctas`: CTAs of the in-switch reduction of a bucket that has the rest of backward to hide under -- few on
        # purpose: a burst of 2 x 128 MiB through the L2 while a GEMM runs evicts the panels that GEMM re-reads (measured
        # on 2 GPUs: the dgrad GEMMs next to a 32-CTA reduction ran 9 ms/step slower); `tail_ctas`: the last buckets of
        # the step, whose reduction is exposed, go at full width
        from alpa_b200 import ops
        self.C = ops.native_module()
        self.offsets = {}
        total = self.FLAG_BYTES
        for p in plans:
            self.offsets[id(p)] = total
            total += (p.numel * 2 + 1023) // 1024 * 1024
        self.ws = SymmWorkspace(group, total)
        if self.ws.multicast_ptr == 0:
            raise RuntimeError("NVLS multicast is not available on this system")
        self.tp, self.rank = self.ws.world, self.ws.rank
        self.flag_ptrs = self.ws.peer_ptrs(0)
        self.counter = torch.zeros(1, dtype=torch.int32, device=self.ws.device)
        from alpa_b200.collective import streams as cstreams
        self.stream = cstreams.comm_stream("grad_reduce")          # one side stream for every gradient reducer
        self.ctas = ctas
        self.tail_ctas = tail_ctas
        self.tail = {id(p) for p in plans[-2:]}

    def bucket(self, comm, plan, logical_mesh):
        from alpa_b200.device_mesh import GradBucket
        if plan.numel % (8 * self.tp):
            raise RuntimeError("bucket size not a multiple of 8 x group size")
        off = self.offsets[id(plan)]
        flat = self.ws.local(off, (plan.numel,), torch.bfloat16)
        arena = self
        ctas = self.tail_ctas if id(plan) in self.tail else self.ctas

        class _NvlsBucket(GradBucket):
            kind = "nvls-multimem"

            def reduce_async(self_inner):
                ev = torch.cuda.Event()
                ev.record(torch.cuda.current_stream())
                with torch.cuda.stream(arena.stream):
                    arena.stream.wait_event(ev)
                    arena.C.peer_barrier_auto(arena.flag_ptrs, arena.counter, arena.rank)
                    arena.C.allreduce_multimem(arena.ws.multicast_ptr + off, plan.numel, arena.rank, arena.tp, ctas)
                    arena.C.peer_barrier_auto(arena.flag_ptrs, arena.counter, arena.rank)
                    done = torch.cuda.Event()
                    done.record(arena.stream)
                return _EventWork(done)

        return _NvlsBucket(comm, plan, logical_mesh, [self.ws.device], flats=[flat])


class _NvlsHandle:
    def __init__(self, reducer, bucket_id):
        self.reducer, self.bucket_id = reducer, bucket_id

    def wait(self):
        self.reducer.wait(self.bucket_id)


class NvlsGradReducer:
    """mode "nvls": in-switch reduction of a symmetric bucket; mode "nccl": the same bucketing in front of one NCCL
    all-reduce per bucket (fewer, larger collectives when multicast memory is unavailable)."""

    def __init__(self, group, bucket_bytes: int = 128 << 20, ctas: int = 24, mode: str = "nvls"):
        from alpa_b200 import ops
        self.mode = mode
        self.group = group
        self.bucket_elems = bucket_bytes // 2
        if mode == "nvls":
            self.C = ops.native_module()
            self.ws = SymmWorkspace(group, 2 * bucket_bytes)
            if self.ws.multicast_ptr == 0:
                raise RuntimeError("NVLS multicast is not available on this system")
            self.tp, self.rank = self.ws.world, self.ws.rank
        else:
            self.ws = None
            self.flat = torch.empty(2 * self.bucket_elems, dtype=torch.bfloat16, device="cuda")
            self.tp, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.ctas = ctas
        from alpa_b200.collective import streams as cstreams
        self.stream = cstreams.comm_stream("grad_reduce")          # one side stream for every gradient reducer
        self.cur = 0                       # bucket being filled (id grows monotonically; slot = id & 1)
        self.fill = 0
        self.items: List[Tuple[torch.Tensor, int, int]] = []
        self.done_events: Dict[int, torch.cuda.Event] = {}
        self.flushed = -1

    def _slot_view(self, bucket_id, off, n):
        base = (bucket_id & 1) * self.bucket_elems
        if self.ws is None:
            return self.flat[base + off:base + off + n]
        return self.ws.local(2 * (base + off), (n,), torch.bfloat16)

    def add(self, t: torch.Tensor) -> Optional[_NvlsHandle]:
        n = t.numel()
        n_pad = (n + 7) // 8 * 8
        if n_pad > self.bucket_elems or t.dtype != torch.bfloat16 or not t.is_contiguous():
            return None
        if self.fill + n_pad > self.bucket_elems:
            self.flush()
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        with torch.cuda.stream(self.stream):
            self.stream.wait_event(ev)
            self._slot_view(self.cur, self.fill, n).copy_(t.view(-1), non_blocking=True)
        t.record_stream(self.stream)
        self.items.append((t, self.fill, n))
        self.fill += n_pad
        return _NvlsHandle(self, self.cur)

    def flush(self):
        if not self.items:
            return
        bid = self.cur
        base = (bid & 1) * self.bucket_elems
        total = (self.fill + 8 * self.tp - 1) // (8 * self.tp) * (8 * self.tp)
        with torch.cuda.stream(self.stream):
            if total > self.fill:
                self._slot_view(bid, self.fill, total - self.fill).zero_()
            if self.ws is None:
                dist.all_reduce(self._slot_view(bid, 0, total), group=self.group)
            else:
                self.ws.barrier()                  # every rank has packed this bucket
                self.C.allreduce_multimem(self.ws.multicast_ptr + 2 * base, total, self.rank, self.tp, self.ctas)
                self.ws.barrier()                  # every slice is reduced and broadcast
            for (t, off, n) in self.items:
                t.view(-1).copy_(self._slot_view(bid, off, n), non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self.done_events[bid] = ev
        self.flushed = bid
        self.items = []
        self.fill = 0
        self.cur += 1

    def wait(self, bucket_id: int):
        if bucket_id > self.flushed:
            self.flush()
        ev = self.done_events.get(bucket_id)
        if ev is not None:
            torch.cuda.current_stream().wait_event(ev)
