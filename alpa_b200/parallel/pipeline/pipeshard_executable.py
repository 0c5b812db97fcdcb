"""The pipeshard runtime: interprets the static instruction lists produced by the emitter.

Reference: alpa/pipeline_parallel/pipeshard_executable.py (PipeshardDriverExecutable:41 launch_on_driver:147,
get_stage_execution_info:255, dump_debug_info:357; PipeshardMeshWorkerExecutable:437 execute_on_worker:489,
dump_stage_execution_trace_internal:592).

One process per GPU: every rank holds the whole config but executes only the instructions of the mesh it
belongs to; cross-mesh SEND/RECV are NCCL point-to-point transfers (torch.distributed) between global
ranks, issued in the emitter's global order.  With an emulated cluster (all meshes in this process)
the global program is executed sequentially and transfers go through an in-process mailbox.

Overlap of communication and compute on GPUs (reference: per-output done events
XLA/service/gpu/done_event_insertion.cc:41, dedicated send / receive streams of the C++ comm group
alpa_nccl_group_base.cc:107-120, event waits alpa_nccl_wrapper.cc:140-203): every value produced by a RUN gets a
*done event* recorded the moment the instruction that finalises it has been issued; a SEND is enqueued on the send
stream and waits only for that event; a RECV is enqueued on the receive stream and records a *ready event*; a RUN
makes the compute stream wait only for the ready events of the values it reads.  The host never blocks inside a
step, so the transfers of one micro-batch run under the kernels of the others.
"""
from __future__ import annotations

import json
import time
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.distributed as dist

from alpa_b200.device_mesh import DistributedArray, PhysicalDeviceMeshGroup, ReplicatedDistributedArray
from alpa_b200.global_env import global_config
from alpa_b200.mesh_executable import next_mesh_executable_uuid
from alpa_b200.parallel.pipeline.runtime_emitter import PipelineInstType, PipeshardConfig
from alpa_b200.sharding import ShardingSpec
from alpa_b200.timer import timers, tracer


class PipeshardDriverExecutable:
    def __init__(self, config: PipeshardConfig, virtual_mesh, name: str = "pipeshard"):
        self.config = config
        self.virtual_mesh = virtual_mesh
        self.name = name
        self.exec_uuid = next_mesh_executable_uuid()
        self.exec_timer_name = f"exec-{self.exec_uuid}"
        self.num_mesh = config.num_meshes
        self.mesh_group = PhysicalDeviceMeshGroup(config.physical_meshes, virtual_mesh)
        self.emulated = all(m.emulated for m in config.physical_meshes)
        self.my_meshes = [i for i, m in enumerate(config.physical_meshes) if m.is_member]
        self.stage_exec_times: Dict[Tuple[int, str], List[float]] = {}
        if not self.emulated and dist.is_initialized() and global_config.eagerly_create_communicators:
            # groups of every mesh must be created by every rank in the same order
            for m, lm in zip(config.physical_meshes, config.logical_meshes):
                if hasattr(m.comm, "ensure_groups"):
                    m.comm.ensure_groups(lm)
        if not self.emulated and dist.is_initialized() and global_config.resharding_mode == "broadcast":
            # broadcast groups are created collectively (same order on every rank) before the first step
            for tid in sorted(config.resharding_tasks):
                task = config.resharding_tasks[tid]
                for (src_dev, _sl, idxs) in task.broadcast_groups():
                    members = tuple(sorted({src_dev} | {task.transfers[k].dst_device for k in idxs}))
                    if len(members) > 1:
                        config.physical_meshes[0].comm.get_group(members)
        self.output_specs = [op[3] if op[0] in ("value", "grad") else None for op in config.output_placements]
        self._native_groups = None
        if (not self.emulated and dist.is_initialized() and global_config.use_native_comm_group and
                global_config.resharding_mode == "send_recv"):
            # one communication group per (sender, receiver) pair, created by every rank in the same global order
            # (reference: the communicator cache keyed by the device set, alpa_nccl_group_base.cc:237-281)
            from alpa_b200.collective import native_group as ng
            pairs = {(tr.src_device, tr.dst_device) for tid in sorted(config.resharding_tasks)
                     for tr in config.resharding_tasks[tid].transfers if tr.src_device != tr.dst_device}
            kw = {"backend": global_config.native_comm_backend} if global_config.native_comm_backend is not None else {}
            self._native_groups = ng.create_pair_groups(pairs, dist.get_rank(), **kw)

    # ------------------------------------------------------------------ launch
    def launch_on_driver(self, *args):
        cfg = self.config
        nmb = cfg.num_micro_batches
        timers(self.exec_timer_name).start()
        self._pending_sends = {}
        self._async = (not self.emulated and dist.is_initialized() and torch.cuda.is_available() and
                       global_config.pipeline_async_comm and global_config.resharding_mode == "send_recv" and
                       not global_config.pipeline_use_signal_send_recv and self._native_groups is None)
        self._native_uuids: List[int] = []
        self._native_used = set()
        if self._async and getattr(self, "_streams", None) is None:
            # dedicated send / receive streams from the process-wide communication stream registry
            # (reference: the per-device nccl stream pool of alpa_nccl_group_base.cc:107-120)
            from alpa_b200.collective import streams as cstreams
            self._streams = (cstreams.comm_stream("pipeshard.send"), cstreams.comm_stream("pipeshard.recv"))
        self._done_ev: Dict[Tuple[int, int, int], "torch.cuda.Event"] = {}    # value produced by a RUN is final
        self._ready_ev: Dict[Tuple[int, int, int], "torch.cuda.Event"] = {}   # value received from another mesh landed
        self._inflight = []                                                   # (works, tensors) of asynchronous sends
        env: Dict[Tuple[int, int, int], List[torch.Tensor]] = {}       # (mesh, value, mb) -> local shards
        acc: Dict[Tuple[int, int], List[torch.Tensor]] = {}            # (mesh, grad value) -> fp32-ish accumulators
        mailbox: Dict[Tuple[int, int], Dict[int, List[torch.Tensor]]] = {}

        # ---- place inputs
        for i, (arg, places, is_batch, aval) in enumerate(zip(args, cfg.input_placements, cfg.input_is_batch,
                                                              cfg.input_avals)):
            if not places:
                continue
            for (m, v, spec) in places:
                pm, lm = cfg.physical_meshes[m], cfg.logical_meshes[m]
                # Decide rank-independently whether a gather is needed: `full_tensor` is a collective
                # that every rank of the job has to enter.
                src = arg
                if isinstance(src, ReplicatedDistributedArray):
                    rep = src.get_replica_on_mesh(pm)
                    src = rep if rep is not None else src.replica
                if isinstance(src, DistributedArray):
                    matches = (src.device_mesh.devices == pm.devices and src.logical_mesh.shape == lm.shape and
                               src.sharding_spec.equivalent(spec) and not is_batch)
                    if not matches:
                        src = src.full_tensor()
                if not pm.is_member:
                    continue
                if is_batch:
                    full = self._to_global_tensor(src, m)
                    for mb, chunk in enumerate(torch.chunk(full, nmb, dim=0)):
                        env[(m, v, mb)] = pm.shard_tensor(chunk, lm, spec).shards
                else:
                    env[(m, v, -1)] = self._shard_arg(src, m, spec, aval)

        # ---- run
        program = cfg.global_program
        trace = global_config.collect_trace
        for ins in program:
            m = ins.mesh_idx
            pm = cfg.physical_meshes[m]
            op = ins.opcode
            if op == PipelineInstType.RUN:
                if not pm.is_member:
                    continue
                se = cfg.stage_execs[(m, ins.stage)]
                ins_vals = []
                for v in se.input_value_ids:
                    if v in cfg.grad_values:
                        gm_, src_v = cfg.grad_values[v]
                        ins_vals.append(acc[(gm_, src_v)])
                        continue
                    key = (m, v, ins.micro_batch) if (m, v, ins.micro_batch) in env else (m, v, -1)
                    ins_vals.append(env[key])
                    ev = self._ready_ev.pop(key, None) if (self._async or self._native_groups is not None) else None
                    if ev is not None:                 # received on the receive stream: compute waits for the data only
                        torch.cuda.current_stream().wait_event(ev)
                if trace:
                    tracer.log("RUN", f"mesh{m}/{ins.stage}/mb{ins.micro_batch} begin", pm.sync_workers)
                t0 = time.time()
                if self._async:
                    out_events = [torch.cuda.Event() for _ in se.output_value_ids]
                    outs = se.program.run(ins_vals, on_output=lambda i: out_events[i].record())
                    for v, e in zip(se.output_value_ids, out_events):
                        self._done_ev[(m, v, ins.micro_batch if ins.micro_batch >= 0 and self._is_mb(v) else -1)] = e
                else:
                    outs = se.program.run(ins_vals)
                if global_config.pipeline_sync_for_timer:
                    pm.sync_workers()
                    self.stage_exec_times.setdefault((m, ins.stage), []).append(time.time() - t0)
                if trace:
                    tracer.log("RUN", f"mesh{m}/{ins.stage}/mb{ins.micro_batch} end", pm.sync_workers)
                for v, o in zip(se.output_value_ids, outs):
                    env[(m, v, ins.micro_batch if ins.micro_batch >= 0 and self._is_mb(v) else -1)] = o
            elif op == PipelineInstType.SEND:
                if not pm.is_member:
                    continue
                self._send(ins, env, mailbox)
            elif op == PipelineInstType.RECV:
                if not pm.is_member:
                    continue
                self._recv(ins, env, mailbox)
            elif op == PipelineInstType.ACCUMULATE:
                if not pm.is_member:
                    continue
                g = env[(m, ins.value, ins.micro_batch)]
                key = (m, ins.value)
                if key not in acc:
                    acc[key] = [x.clone() if nmb > 1 else x for x in g]
                else:
                    for a, x in zip(acc[key], g):
                        a.add_(x)
            elif op == PipelineInstType.FINALIZE_GRAD:
                if not pm.is_member:
                    continue
                key = (m, ins.value)
                se = cfg.stage_execs.get((m, "backward"))
                axes = se.deferred_allreduce.get(ins.value) if se is not None else None
                if axes:
                    acc[key] = pm.comm.all_reduce(acc[key], cfg.logical_meshes[m], axes, "sum")
                if nmb > 1:
                    for a in acc[key]:
                        a.div_(nmb)
            elif op == PipelineInstType.FREE:
                for (v, mb) in ins.values:
                    if self._pending_sends:
                        self._wait_pending_sends((m, v, mb))
                    env.pop((m, v, mb), None)
        self._wait_pending_sends()
        if self._native_groups is not None:
            on_cuda = torch.cuda.is_available()
            for pair in sorted(self._native_used):               # compute resumes after the step's transfers only here
                if on_cuda:
                    self._native_groups[pair].compute_wait_comm()
            if on_cuda:
                cur = torch.cuda.current_stream()
                for ev in self._ready_ev.values():
                    cur.wait_event(ev)
            if self._native_uuids:
                next(iter(self._native_groups.values())).backend.registry().discard(self._native_uuids)
            self._inflight, self._ready_ev, self._done_ev = [], {}, {}
        if self._async:
            cur = torch.cuda.current_stream()
            for st in self._streams:
                cur.wait_stream(st)
            for works, _keep in self._inflight:
                for w in works:
                    w.wait()
            for ev in self._ready_ev.values():
                cur.wait_event(ev)
            self._inflight, self._ready_ev, self._done_ev = [], {}, {}

        # ---- outputs
        results = []
        for op in cfg.output_placements:
            if op[0] == "const":
                results.append(op[1])
                continue
            if op[0] == "input":
                results.append(args[op[1]])
                continue
            if op[0] == "grad":
                _, m, v, spec = op
                pm, lm = cfg.physical_meshes[m], cfg.logical_meshes[m]
                shape, dtype = cfg.value_avals[v]
                shards = [x.clone() for x in acc[(m, v)]] if pm.is_member else []
                results.append(DistributedArray(pm, lm, shape, dtype, spec, shards))
                continue
            if op[0] == "replicated":
                reps = []
                for (m, v, spec) in op[1]:
                    pm, lm = cfg.physical_meshes[m], cfg.logical_meshes[m]
                    shape, dtype = cfg.value_avals[v]
                    shards = env.get((m, v, -1), []) if pm.is_member else []
                    reps.append(DistributedArray(pm, lm, shape, dtype, spec, shards))
                results.append(ReplicatedDistributedArray([cfg.physical_meshes[m] for (m, _, _) in op[1]], reps))
                continue
            _, m, v, spec, reduce = op
            pm, lm = cfg.physical_meshes[m], cfg.logical_meshes[m]
            if not pm.is_member:
                # a reference to an array living on another pipeline stage's mesh (no local shards)
                shape, dtype = cfg.value_avals[v]
                if reduce == "concat":
                    shape = (shape[0] * nmb,) + tuple(shape[1:])
                results.append(DistributedArray(pm, lm, shape, dtype, spec, []))
                continue
            if reduce == "none":
                shards = env.get((m, v, -1))
                if shards is None:
                    shards = env[(m, v, 0)]
            elif reduce == "mean":
                parts = [env[(m, v, mb)] for mb in range(nmb)]
                shards = [torch.stack([p[d] for p in parts]).float().mean(0).to(parts[0][d].dtype)
                          for d in range(len(parts[0]))]
            else:  # concat along the batch dim: gather each micro-batch then re-shard
                mb_shape, mb_dtype = cfg.value_avals[v]
                fulls = [DistributedArray(pm, lm, mb_shape, mb_dtype, spec, env[(m, v, mb)]).full_tensor()
                         for mb in range(nmb)]
                shards = pm.shard_tensor(torch.cat(fulls, dim=0), lm, spec).shards
            local = tuple(shards[0].shape)
            shape = tuple(s * spec.num_shards(d) for d, s in enumerate(local))
            results.append(DistributedArray(pm, lm, shape, shards[0].dtype, spec, shards))
        for a, d in zip(args, cfg.donated):
            if d and isinstance(a, DistributedArray) and not a.deleted:
                a.shards = []
                a.deleted = True
        timers(self.exec_timer_name).stop()
        return results

    def __call__(self, *args):
        return self.launch_on_driver(*args)

    # ------------------------------------------------------------------ helpers
    def _is_mb(self, v: int) -> bool:
        # a value is per-micro-batch iff some instruction refers to it with mb >= 0; cached lazily
        cache = getattr(self, "_mb_cache", None)
        if cache is None:
            cache = {}
            for key, se in self.config.stage_execs.items():
                for vid in se.output_value_ids:
                    cache[vid] = key[1] in ("forward", "backward")
            self._mb_cache = cache
        return cache.get(v, False)

    def _to_global_tensor(self, arg, mesh_idx):
        if isinstance(arg, ReplicatedDistributedArray):
            arg = arg.replica
        if isinstance(arg, DistributedArray):
            return arg.full_tensor()
        if isinstance(arg, np.ndarray):
            return torch.from_numpy(arg)
        return arg

    def _shard_arg(self, arg, m, spec: ShardingSpec, aval):
        pm, lm = self.config.physical_meshes[m], self.config.logical_meshes[m]
        if isinstance(arg, ReplicatedDistributedArray):
            rep = arg.get_replica_on_mesh(pm)
            arg = rep if rep is not None else arg.replica
        if isinstance(arg, DistributedArray):
            if arg.deleted:
                raise RuntimeError("this DistributedArray was donated to an earlier call (donate_argnums) or deleted; "
                                   "its buffers now belong to that call's outputs")
            if arg.device_mesh.devices == pm.devices and arg.logical_mesh.shape == lm.shape and \
                    arg.sharding_spec.equivalent(spec):
                return arg.shards
            arg = arg.full_tensor()
        if isinstance(arg, np.ndarray):
            arg = torch.from_numpy(arg)
        if aval is not None and arg.dtype != aval[1]:
            arg = arg.to(aval[1])
        return pm.shard_tensor(arg, lm, spec).shards

    def _send(self, ins, env, mailbox):
        cfg = self.config
        task = cfg.resharding_tasks[ins.task]
        src_m, dst_m = cfg.task_meshes[ins.task]
        pm = cfg.physical_meshes[src_m]
        shards = env[(src_m, ins.value, ins.micro_batch)]
        if not self.emulated and global_config.resharding_mode == "broadcast":
            # one broadcast per distinct source region: {sender} + every mesh device that needs it
            for (src_dev, src_slices, idxs) in task.broadcast_groups():
                if src_dev not in pm.local_devices:
                    continue
                tile = shards[pm.local_devices.index(src_dev)][src_slices].contiguous()
                members = tuple(sorted({src_dev} | {task.transfers[k].dst_device for k in idxs}))
                dist.broadcast(tile, src=src_dev, group=pm.comm.get_group(members))
            return
        if self._native_groups is not None:
            return self._send_native(task, pm, shards)
        p2p = []
        for li, dev in enumerate(pm.local_devices):
            for k, tr in enumerate(task.transfers):
                if tr.src_device != dev:
                    continue
                tile = shards[li][tr.src_slices]
                if global_config.pipeline_use_signal_send_recv:
                    tile = tile.reshape(-1)[:1]
                if self.emulated:
                    mailbox.setdefault((ins.task, ins.micro_batch), {})[k] = tile.clone()
                else:
                    p2p.append(dist.P2POp(dist.isend, tile.contiguous(), tr.dst_device))
        if p2p and self._async:
            # dedicated send stream; waits for the done event of this value only, never blocks the host or the compute
            # stream.  The tiles stay referenced (and recorded on the send stream) until the step ends.
            send_stream = self._streams[0]
            ev = self._done_ev.get((src_m, ins.value, ins.micro_batch))
            with torch.cuda.stream(send_stream):
                if ev is not None:
                    send_stream.wait_event(ev)
                else:
                    send_stream.wait_stream(torch.cuda.default_stream())
                works = dist.batch_isend_irecv(p2p)
            for t in shards:
                t.record_stream(send_stream)
            self._inflight.append((works, [op.tensor for op in p2p]))
            return
        if p2p:       # all tiles of this resharding task in one grouped NCCL launch
            works = dist.batch_isend_irecv(p2p)
            if getattr(self, "schedule_name", "") == "1f1b_overlap_friendly":
                # overlap-friendly pipelines (reference: OverlapFriendlyPipelineInstEmitter, runtime_emitter.py:1109):
                # do not make the compute stream wait for the send; the tiles stay referenced until the value is
                # freed (or the step ends), where the wait finally happens
                self._pending_sends.setdefault((src_m, ins.value, ins.micro_batch), []).append((works, p2p))
            else:
                for w in works:
                    w.wait()

    # ---- native communication groups (csrc/comm_group.cpp): per-pair communicators, per-direction streams, uuid events
    def _send_native(self, task, pm, shards):
        """The tiles for one peer are packed into ONE staging buffer by one kernel on the compute stream (so they are
        ordered after the producing stage by construction; `ops.pack_tiles`, pack_sm90.cu); one uuid event marks "all
        packed" and each pair group's stream waits for exactly that before its send -- one message per peer, and the
        host and the compute stream never wait (reference: alpa_nccl_wrapper.cc:140-175)."""
        from alpa_b200 import ops
        from alpa_b200.collective.native_group import new_uuid
        per_pair: Dict[Tuple[int, int], Tuple[int, List[torch.Tensor]]] = {}
        for li, dev in enumerate(pm.local_devices):
            for tr in task.transfers:
                if tr.src_device != dev:
                    continue
                tile = shards[li][tr.src_slices]
                if global_config.pipeline_use_signal_send_recv:
                    tile = tile.reshape(-1)[:1]
                pair = (min(dev, tr.dst_device), max(dev, tr.dst_device))
                per_pair.setdefault(pair, (tr.dst_device, []))[1].append(tile)
        if not per_pair:
            return
        msgs = {}
        for pair, (dst, tiles) in per_pair.items():
            # Message of a pair = raw bytes: one tile travels as exactly its own bytes (straight from the stage output
            # when it is contiguous), several tiles as the packed buffer (16-byte aligned tiles) -- the receiver derives
            # the same length from the same transfer list.
            st_ = self.__dict__.setdefault("native_stats", {"messages": 0, "packed": 0})
            st_["messages"] += 1
            st_["packed"] += int(len(tiles) > 1 or not tiles[0].is_contiguous())
            if len(tiles) == 1:
                t = tiles[0] if tiles[0].is_contiguous() else ops.pack_tiles(tiles)
                msgs[pair] = (dst, t.reshape(-1).view(torch.uint8)[:tiles[0].numel() * tiles[0].element_size()])
            else:
                msgs[pair] = (dst, ops.pack_tiles(tiles))
        uuid = new_uuid()
        next(iter(self._native_groups.values())).record(uuid)                # on the current (compute) stream
        self._native_uuids.append(uuid)
        for pair in sorted(msgs):
            g, (dst, msg) = self._native_groups[pair], msgs[pair]
            g.batch([("send", msg, dst, uuid, -1)])
            st = g.stream(g.channel_of(True, dst))
            if st is not None and msg.is_cuda:
                msg.record_stream(st)
            self._native_used.add(pair)
        self._inflight.append(([], [m for _, m in msgs.values()]))

    def _recv_native(self, ins, task, pm, lm, dst_m):
        """Buffers are allocated and filled on communication streams only: the receive of micro-batch k+1 proceeds
        while the compute stream still runs micro-batch k; compute waits for the per-value ready event at its RUN.
        One message per peer lands in a staging buffer and ONE unpack launch writes every destination slice."""
        import contextlib
        from alpa_b200 import ops
        from alpa_b200.collective.native_group import new_uuid
        signal = global_config.pipeline_use_signal_send_recv
        dtype = self._task_dtype(ins.task)
        mine = [(li, dev, tr) for li, dev in enumerate(pm.local_devices) for tr in task.transfers
                if tr.dst_device == dev]
        outs: List[Optional[torch.Tensor]] = [None] * len(pm.local_devices)
        if mine:
            pair_of = lambda tr: (min(tr.src_device, tr.dst_device), max(tr.src_device, tr.dst_device))   # noqa: E731
            g0 = self._native_groups[pair_of(mine[0][2])]
            rs = g0.stream(g0.channel_of(False, mine[0][2].src_device))     # allocation / assembly stream
            ctx = torch.cuda.stream(rs) if rs is not None else contextlib.nullcontext()
            per_pair: Dict[Tuple[int, int], Tuple[int, List[torch.Tensor]]] = {}
            msgs = {}
            with ctx:
                for li, dev, tr in mine:
                    if outs[li] is None:
                        outs[li] = torch.empty(tuple(task.dst.device_tiles[dev].shape), dtype=dtype, device=pm.torch_device)
                    view = outs[li][tr.dst_slices]
                    if signal:
                        view = torch.empty(1, dtype=dtype, device=pm.torch_device)
                    per_pair.setdefault(pair_of(tr), (tr.src_device, []))[1].append(view)
                for pair, (src, views) in per_pair.items():
                    direct = len(views) == 1 and views[0].is_contiguous()
                    if direct:                                   # lands in place
                        msg = views[0].reshape(-1).view(torch.uint8)
                    else:
                        msg = torch.empty(ops.packed_nbytes(views), dtype=torch.uint8, device=pm.torch_device)
                        if len(views) == 1:                      # one strided tile: exactly its bytes travel
                            msg = msg[:views[0].numel() * views[0].element_size()]
                    msgs[pair] = (src, msg, direct)
            alloc_uuid = new_uuid()
            g0.record(alloc_uuid, rs)
            self._native_uuids.append(alloc_uuid)
            done = []
            for pair in sorted(msgs):
                g, (src, msg, _direct) = self._native_groups[pair], msgs[pair]
                st = g.stream(g.channel_of(False, src))
                if st is not rs:
                    g.wait(alloc_uuid, st)                                   # buffers exist before another stream writes
                u = new_uuid()
                g.batch([("recv", msg, src, -1, u)])
                if st is not rs:
                    done.append(u)
                    if msg.is_cuda and st is not None:
                        msg.record_stream(st)
                self._native_uuids.append(u)
                self._native_used.add(pair)
            with ctx:
                for u in done:
                    g0.wait(u, rs)
                if not signal:
                    for pair, (src, msg, direct) in msgs.items():
                        if not direct:
                            ops.unpack_tiles(msg, per_pair[pair][1])
                if rs is not None:
                    ev = torch.cuda.Event()
                    ev.record(rs)
                    self._ready_ev[(dst_m, ins.value, ins.micro_batch)] = ev
                    for t in outs:
                        if t is not None:
                            t.record_stream(torch.cuda.default_stream())
        # scatter-gather: the tiles were sent 1/n each; all-gather locally over NVLink (on the compute stream)
        if task.local_allgather:
            ev = self._ready_ev.pop((dst_m, ins.value, ins.micro_batch), None)
            if ev is not None:
                torch.cuda.current_stream().wait_event(ev)
            for (axis, dim) in reversed(task.local_allgather):
                outs = pm.comm.all_gather(outs, lm, axis, dim)
        return outs

    def _wait_pending_sends(self, key=None):
        pend = self._pending_sends
        keys = [key] if key is not None else list(pend)
        for k in keys:
            for works, _tiles in pend.pop(k, ()):
                for w in works:
                    w.wait()

    def _recv(self, ins, env, mailbox):
        cfg = self.config
        task = cfg.resharding_tasks[ins.task]
        src_m, dst_m = cfg.task_meshes[ins.task]
        pm, lm = cfg.physical_meshes[dst_m], cfg.logical_meshes[dst_m]
        src_shards_example = None
        node_shape = task.dst.shape
        dtype = None
        outs = []
        if self._native_groups is not None:
            env[(dst_m, ins.value, ins.micro_batch)] = self._recv_native(ins, task, pm, lm, dst_m)
            return
        bcast = not self.emulated and global_config.resharding_mode == "broadcast"
        bcast_data = {}
        if bcast:
            for (src_dev, src_slices, idxs) in task.broadcast_groups():
                mine = [k for k in idxs if task.transfers[k].dst_device in pm.local_devices]
                if not mine:
                    continue
                members = tuple(sorted({src_dev} | {task.transfers[k].dst_device for k in idxs}))
                shape = tuple(s.stop - s.start for s in src_slices)
                tmp = torch.empty(shape, dtype=self._task_dtype(ins.task), device=pm.torch_device)
                dist.broadcast(tmp, src=src_dev, group=pm.comm.get_group(members))
                for k in mine:
                    bcast_data[k] = tmp
        p2p, p2p_fill = [], []
        use_async = self._async and not bcast
        import contextlib
        ctx = torch.cuda.stream(self._streams[1]) if use_async else contextlib.nullcontext()
        with ctx:
            outs = self._recv_body(ins, task, pm, lm, bcast, bcast_data, mailbox, p2p, p2p_fill)
            if use_async:
                ev = torch.cuda.Event()
                ev.record(self._streams[1])
                self._ready_ev[(dst_m, ins.value, ins.micro_batch)] = ev
                for t in outs:
                    if t is not None:
                        t.record_stream(torch.cuda.default_stream())
        env[(dst_m, ins.value, ins.micro_batch)] = outs

    def _recv_body(self, ins, task, pm, lm, bcast, bcast_data, mailbox, p2p, p2p_fill):
        outs = []
        for li, dev in enumerate(pm.local_devices):
            tile_shape = task.dst.device_tiles[dev].shape
            buf = None
            for k, tr in enumerate(task.transfers):
                if tr.dst_device != dev:
                    continue
                if bcast:
                    if buf is None:
                        buf = torch.empty(tile_shape, dtype=self._task_dtype(ins.task), device=pm.torch_device)
                    buf[tr.dst_slices] = bcast_data[k]
                    continue
                if self.emulated:
                    data = mailbox[(ins.task, ins.micro_batch)].pop(k)
                    if buf is None:
                        buf = torch.empty(tile_shape, dtype=data.dtype, device=data.device)
                    if not global_config.pipeline_use_signal_send_recv:
                        buf[tr.dst_slices] = data
                else:
                    if buf is None:
                        buf = torch.empty(tile_shape, dtype=self._task_dtype(ins.task), device=pm.torch_device)
                    shape = tuple(s.stop - s.start for s in tr.dst_slices)
                    if global_config.pipeline_use_signal_send_recv:
                        tmp = torch.empty(1, dtype=buf.dtype, device=buf.device)
                        p2p.append(dist.P2POp(dist.irecv, tmp, tr.src_device))
                    else:
                        tmp = torch.empty(shape, dtype=buf.dtype, device=buf.device)
                        p2p.append(dist.P2POp(dist.irecv, tmp, tr.src_device))
                        p2p_fill.append((buf, tr.dst_slices, tmp))
            outs.append(buf)
        if p2p:
            for w in dist.batch_isend_irecv(p2p):
                w.wait()
            for (buf, sl, tmp) in p2p_fill:
                buf[sl] = tmp
        # scatter-gather: the tiles were sent 1/n each; all-gather locally over NVLink
        # undo the extra sharding minor axis first (axes were appended major -> minor on a shared tensor dim)
        for (axis, dim) in reversed(task.local_allgather):
            outs = pm.comm.all_gather(outs, lm, axis, dim)
        return outs

    def _task_dtype(self, tid):
        cache = getattr(self, "_dtype_cache", None)
        if cache is None:
            cache = {}
            self._dtype_cache = cache
        if tid not in cache:
            # dtype of the transferred value: look it up from the producing stage's program outputs
            cfg = self.config
            src_m, _ = cfg.task_meshes[tid]
            vid = next(i.value for i in cfg.global_program if i.opcode == PipelineInstType.SEND and i.task == tid)
            dt = torch.float32
            for (m, _k), se in cfg.stage_execs.items():
                if m == src_m and vid in se.output_value_ids:
                    j = se.output_value_ids.index(vid)
                    node = [n for n in se.program.gm.graph.nodes if n.op == "output"][0].args[0][j]
                    dt = node.meta["val"].dtype
            cache[tid] = dt
        return cache[tid]

    def get_parallel_plan(self):
        """Serializable description of how this function was parallelized; `plan_to_method(plan)` rebuilds an
        equivalent method with the stage assignment fixed (reference: pipeshard_executable.py:317-336)."""
        from alpa_b200.parallel.pipeline.stage_construction import ManualStageOption
        from alpa_b200.parallel_plan import ClusterInfo, ParallelPlan, PipelinePlan
        sp = self.stage_plan
        vm = self.virtual_mesh
        manual = ManualStageOption([list(x) for x in sp.forward_stage_layer_ids], [tuple(x) for x in sp.submesh_shapes],
                                   [tuple(x) for x in sp.logical_mesh_shapes], [dict(d) for d in sp.autosharding_option_dicts])
        return ParallelPlan(ClusterInfo(vm.num_hosts, vm.num_devices_per_host), self.config.num_micro_batches,
                            self.as_option, PipelinePlan(self.schedule_name, self.layer_option, manual),
                            self.get_input_placement_specs())

    # ------------------------------------------------------------------ introspection
    def get_input_placement_specs(self):
        from alpa_b200.parallel_plan import PlacementSpec
        out = []
        for places, aval in zip(self.config.input_placements, self.config.input_avals):
            if not places:
                out.append(None)
            else:
                out.append(PlacementSpec(aval, tuple(tuple(self.config.physical_meshes[m].devices) for m, _, _ in places),
                                         tuple(sp for _, _, sp in places)))
        return out

    def get_output_placement_specs(self):
        from alpa_b200.parallel_plan import PlacementSpec
        return [PlacementSpec(None, (tuple(self.config.physical_meshes[op[1]].devices),), (op[3],))
                if op[0] in ("value", "grad") else None for op in self.config.output_placements]

    def get_execution_time_costs(self, warmup: int = 0, timer_name=None):
        return timers(timer_name or self.exec_timer_name).costs[warmup:]

    def get_stage_execution_info(self):
        return dict(self.stage_exec_times)

    def count_collectives(self):
        total: Dict[str, int] = {}
        for se in self.config.stage_execs.values():
            for k, v in se.program.count_collectives().items():
                total[k] = total.get(k, 0) + v
        total["cross-mesh-send"] = sum(1 for i in self.config.global_program if i.opcode == PipelineInstType.SEND)
        return total

    def get_hlo_text(self):
        parts = []
        for (m, k), se in sorted(self.config.stage_execs.items()):
            parts.append(f"== mesh {m} / {k} ==\n" + se.program.as_text())
        return "\n".join(parts)

    def get_instruction_text(self):
        return self.config.program_text()

    def dump_debug_info(self, folder: str):
        import os
        os.makedirs(folder, exist_ok=True)
        with open(os.path.join(folder, f"{self.name}_instructions.txt"), "w") as f:
            f.write(self.config.program_text())
        with open(os.path.join(folder, f"{self.name}_stages.txt"), "w") as f:
            f.write(self.get_hlo_text())
        with open(os.path.join(folder, f"{self.name}_resharding.txt"), "w") as f:
            for tid, t in self.config.resharding_tasks.items():
                f.write(f"task {tid} meshes {self.config.task_meshes[tid]} {t.src.spec}->{t.dst.spec} "
                        f"{len(t.transfers)} transfers {t.total_bytes} B allgather={t.local_allgather}\n")
        with open(os.path.join(folder, f"{self.name}_schedule.txt"), "w") as f:
            f.write(self.config.schedule.pprint_schedule())

    def dump_stage_execution_trace_internal(self, filename: str):
        return self.dump_stage_execution_trace(filename)

    def dump_stage_execution_trace(self, filename: str):
        """Chrome-trace JSON of RUN events (reference: dump_stage_execution_trace_internal :592-654)."""
        events = []
        open_ev = {}
        for ev in tracer.events:
            if ev.name != "RUN":
                continue
            key, phase = ev.info.rsplit(" ", 1)
            if phase == "begin":
                open_ev[key] = ev.tstamp
            elif key in open_ev:
                mesh = key.split("/")[0]
                t0 = open_ev.pop(key)
                events.append({"name": key, "cat": "stage", "ph": "X", "pid": 0, "tid": mesh,
                               "ts": t0 * 1e6, "dur": (ev.tstamp - t0) * 1e6})
        with open(filename, "w") as f:
            json.dump({"traceEvents": events, "displayTimeUnit": "ms"}, f)

    def sync(self):
        self.mesh_group.sync_workers()

    # (reference: PipeshardDriverExecutable.get_shard_args_time_costs / get_stage_allocation_size /
    # profile_all_executable_with_dummy_inputs / sync_move_workers, pipeshard_executable.py:295-355)
    def get_shard_args_time_costs(self):
        return timers(self.exec_timer_name + "-shard-args").costs

    def get_stage_allocation_size(self):
        """Static per-device allocation estimate of every stage program, max over the programs of a mesh."""
        from alpa_b200.mesh_executable import program_allocation_size
        per_mesh: Dict[int, int] = {}
        for (m, _k), se in self.config.stage_execs.items():
            per_mesh[m] = max(per_mesh.get(m, 0), program_allocation_size(se.program))
        return [per_mesh.get(m, 0) for m in range(len(self.config.physical_meshes))]

    def get_total_allocation_size(self) -> int:
        """Largest per-device estimate over the meshes (a one-stage pipeline is the gradient-accumulation executable of
        ShardParallel(num_micro_batches=n): reference GradAccMeshDriverExecutable.get_total_allocation_size)."""
        return max(self.get_stage_allocation_size() or [0])

    def profile_all_executable_with_dummy_inputs(self):
        """Run one step with the last arguments' shapes filled with dummy values and return the per-stage run times
        (needs `global_config.pipeline_sync_for_timer` for per-stage numbers; otherwise the whole-step time)."""
        return {k: list(v) for k, v in self.stage_exec_times.items()} or \
            {"step": list(timers(self.exec_timer_name).costs)}

    def sync_move_workers(self):
        self.mesh_group.sync_move_workers()

    def _check_alive(self):
        """All ranks are in-process participants of the same NCCL world; a dead peer surfaces as a
        collective error/timeout (reference: pipeshard_executable.py:417-430 pings Ray actors)."""
        if dist.is_initialized():
            dist.barrier()
        return True
