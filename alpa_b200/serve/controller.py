"""Multi-model serving controller: model registry, replica placement on device-mesh groups, round-robin dispatch,
ASGI/HTTP front end.

Reference: alpa/serve/controller.py (DeviceMeshGroupManager:59 -- one Ray actor per mesh group that hosts model
replicas; Controller:96 -- register_model:132, create_replica:149, handle_asgi:168 picks a replica round-robin and
forwards the request; run_controller:280 starts uvicorn), alpa/serve/http_util.py (ASGI receive/response plumbing),
alpa/serve/run.py.

H100 design: no actor framework.  A mesh group is a set of ranks of the torchrun world; the controller lives on rank
0 of the node and calls replicas in-process (single-GPU models) or broadcasts the request to the ranks of the
replica's tensor-parallel group (`SpmdReplica`), which all execute the same `handle_request`.  The HTTP side is a
plain ASGI application (served by uvicorn when launched through `run_controller`).
"""
from __future__ import annotations

import asyncio
import dataclasses
import json
import logging
import threading
import time
from typing import Any, Callable, Dict, List, Optional, Sequence

logger = logging.getLogger(__name__)

CONTROLLER_NAME = "controller"
MAX_REPLICA_FAILURE_RETRIES = 10


@dataclasses.dataclass
class CreateInfo:
    model_def: Callable
    init_args: Sequence[Any]
    init_kwargs: Dict[str, Any]

    def append_init_args(self, init_args: Optional[Sequence[Any]] = None, init_kwargs: Optional[Dict[str, Any]] = None):
        return CreateInfo(self.model_def, tuple(self.init_args) + tuple(init_args or ()),
                          {**self.init_kwargs, **(init_kwargs or {})})


@dataclasses.dataclass
class ModelInfo:
    create_info: CreateInfo
    managers: List["DeviceMeshGroupManager"]
    next_pt: int = 0


class DeviceMeshGroupManager:
    """Hosts the model replicas placed on one group of device meshes (reference: controller.py:59-93)."""

    def __init__(self, mesh_group_id: int, virtual_mesh_shape: Optional[Sequence[int]] = None, devices=None):
        self.mesh_group_id = mesh_group_id
        self.virtual_mesh_shape = tuple(virtual_mesh_shape) if virtual_mesh_shape else None
        self.devices = devices
        self.replicas: Dict[str, Any] = {}

    def create_replica(self, name: str, create_info: CreateInfo):
        assert name not in self.replicas, f"replica of {name} already exists on mesh group {self.mesh_group_id}"
        self.replicas[name] = create_info.model_def(*create_info.init_args, **create_info.init_kwargs)

    def delete_replica(self, name: str):
        self.replicas.pop(name, None)

    async def handle_request(self, name: str, request: "Request"):
        replica = self.replicas[name]
        fn = getattr(replica, "handle_request", replica)
        out = fn(request)
        if asyncio.iscoroutine(out):
            out = await out
        return out


class Request:
    """Minimal request object handed to replicas (reference: starlette Request built in http_util.py)."""

    def __init__(self, scope: Dict, body: bytes):
        self.scope = scope
        self.method = scope.get("method", "POST")
        self.path = scope.get("path", "/")
        self.query_string = scope.get("query_string", b"").decode()
        self._body = body

    def body(self) -> bytes:
        return self._body

    def json(self) -> Any:
        return json.loads(self._body.decode() or "{}")


class Controller:
    """(reference: Controller, controller.py:96-277)"""

    def __init__(self, host: str = "127.0.0.1", port: int = 20001, root_path: str = "/"):
        self.host, self.port, self.root_path = host, port, root_path
        self.manager_lock: Dict[Any, asyncio.Lock] = {}
        self.mesh_group_managers: Dict[int, DeviceMeshGroupManager] = {}
        self.model_info: Dict[str, ModelInfo] = {}
        self._server = None
        self._thread: Optional[threading.Thread] = None

    # ---- cluster / models
    def launch_mesh_group_manager(self, group_id: int, virtual_mesh_shape=None, devices=None):
        assert group_id not in self.mesh_group_managers, f"Mesh group {group_id} is already launched"
        self.mesh_group_managers[group_id] = DeviceMeshGroupManager(group_id, virtual_mesh_shape, devices)

    def register_model(self, name: str, model_def: Callable, init_args: Optional[Sequence[Any]] = None,
                       init_kwargs: Optional[Dict[str, Any]] = None, override: bool = False):
        if name in self.model_info:
            if not override:
                raise ValueError(f"Model {name} is already registered")
            for m in self.model_info[name].managers:
                m.delete_replica(name)
        self.model_info[name] = ModelInfo(CreateInfo(model_def, tuple(init_args or ()), dict(init_kwargs or {})), [])

    def delete_model(self, name: str):
        info = self.model_info.pop(name, None)
        if info is not None:
            for m in info.managers:
                m.delete_replica(name)

    def create_replica(self, name: str, mesh_group_id: int, append_init_args=None, append_init_kwargs=None):
        assert mesh_group_id in self.mesh_group_managers, f"Group {mesh_group_id} does not exist"
        info = self.model_info[name]
        manager = self.mesh_group_managers[mesh_group_id]
        assert manager not in info.managers
        manager.create_replica(name, info.create_info.append_init_args(append_init_args, append_init_kwargs))
        info.managers.append(manager)

    def list_models(self) -> Dict[str, int]:
        return {k: len(v.managers) for k, v in self.model_info.items()}

    # ---- request path
    async def handle_request(self, name: str, request: Request):
        if name not in self.model_info:
            raise KeyError(f"Model {name} is not registered")
        info = self.model_info[name]
        if not info.managers:
            raise RuntimeError(f"No replica of {name} is created")
        manager = info.managers[info.next_pt]                       # round robin (reference: controller.py:196-199)
        info.next_pt = (info.next_pt + 1) % len(info.managers)
        return await manager.handle_request(name, request)

    async def handle_asgi(self, scope, receive, send):
        """ASGI entry (reference: handle_asgi, controller.py:168-217): body JSON must carry {"model": name}."""
        if scope["type"] == "lifespan":
            while True:
                msg = await receive()
                if msg["type"] == "lifespan.startup":
                    await send({"type": "lifespan.startup.complete"})
                elif msg["type"] == "lifespan.shutdown":
                    await send({"type": "lifespan.shutdown.complete"})
                    return
        assert scope["type"] == "http"
        body = b""
        while True:
            msg = await receive()
            body += msg.get("body", b"")
            if not msg.get("more_body"):
                break
        status, payload = 200, None
        try:
            if scope.get("path", "/").rstrip("/").endswith("/models") and scope.get("method") == "GET":
                payload = self.list_models()
            else:
                request = Request(scope, body)
                obj = request.json()
                name = obj.get("model") if isinstance(obj, dict) else None
                if name is None:
                    status, payload = 400, {"type": "error", "message": "the request body needs a 'model' field"}
                else:
                    payload = await self.handle_request(name, request)
        except KeyError as e:
            status, payload = 404, {"type": "error", "message": str(e)}
        except Exception as e:  # noqa: BLE001
            logger.exception("request failed")
            status, payload = 500, {"type": "error", "message": f"{type(e).__name__}: {e}"}
        from alpa_b200.serve.http_util import _json_default
        data = payload if isinstance(payload, (bytes, bytearray)) else json.dumps(payload, default=_json_default).encode()
        await send({"type": "http.response.start", "status": status,
                    "headers": [(b"content-type", b"application/json"), (b"content-length", str(len(data)).encode())]})
        await send({"type": "http.response.body", "body": bytes(data)})

    async def __call__(self, scope, receive, send):
        await self.handle_asgi(scope, receive, send)

    # ---- http server
    def run_http_server(self, block: bool = False):
        import uvicorn
        config = uvicorn.Config(self, host=self.host, port=self.port, log_level="warning", lifespan="on")
        self._server = uvicorn.Server(config)
        if block:
            self._server.run()
            return
        self._thread = threading.Thread(target=self._server.run, daemon=True)
        self._thread.start()
        for _ in range(100):
            if getattr(self._server, "started", False):
                break
            time.sleep(0.05)

    def get_info(self) -> Dict[str, Any]:
        """(reference: Controller.get_info, controller.py:208-213)"""
        return {"host": self.host, "port": self.port, "root_path": self.root_path}

    async def ready(self, timeout: float = 10.0) -> bool:
        """Returns once the HTTP server accepts traffic; raises if it failed to start (reference: Controller.ready)."""
        t0 = time.time()
        while time.time() - t0 < timeout:
            if self._server is not None and getattr(self._server, "started", False):
                return True
            if self._thread is not None and not self._thread.is_alive():
                raise RuntimeError("the HTTP server thread exited before it was ready")
            await asyncio.sleep(0.02)
        raise TimeoutError(f"the HTTP server was not ready after {timeout} s")

    def shutdown(self):
        if self._server is not None:
            self._server.should_exit = True
        if self._thread is not None:
            self._thread.join(timeout=5)
        for info in self.model_info.values():
            for m in info.managers:
                m.replicas.clear()


def run_controller(host: str = "127.0.0.1", port: int = 20001, root_path: str = "/", block: bool = False) -> Controller:
    """Start the controller and its HTTP server (reference: run_controller, controller.py:280-299)."""
    controller = Controller(host, port, root_path)
    controller.run_http_server(block=block)
    return controller


class SpmdReplica:
    """Replica whose model spans a tensor-parallel group: rank 0 receives the request from the controller and
    broadcasts it; every rank of the group runs `fn(request_obj)` (the collectives inside need all of them)."""

    def __init__(self, fn: Callable[[Any], Any], group=None):
        self.fn = fn
        self.group = group

    def handle_request(self, request: Request):
        import torch.distributed as dist
        obj = request.json()
        if self.group is not None and dist.is_initialized():
            box = [obj]
            dist.broadcast_object_list(box, src=dist.get_global_rank(self.group, 0) if hasattr(dist, "get_global_rank")
                                       else 0, group=self.group)
        return self.fn(obj)

    def worker_loop(self):
        """Run on the non-zero ranks of the group: wait for broadcast requests until None arrives."""
        import torch.distributed as dist
        while True:
            box = [None]
            dist.broadcast_object_list(box, src=dist.get_global_rank(self.group, 0) if hasattr(dist, "get_global_rank")
                                       else 0, group=self.group)
            if box[0] is None:
                return
            self.fn(box[0])
