"""alpa_b200.ops -- the primitive operator set of the framework.

Every primitive is a ``torch.library`` custom op in the ``alpa_b200`` namespace with

* a CUDA/bf16 implementation backed by the hand-written sm_90a kernels in ``ops/csrc`` (``_C``),
* a plain PyTorch reference implementation of the same maths (CPU, fp32, and the numerics oracle),
* a fake (meta) implementation so train steps can be traced without touching a device,
* an autograd formula expressed in other primitives (so fwd+bwd trace to one flat graph), and
* a sharding signature used by the auto-sharding planner (``alpa_b200/parallel/shard``).

Every op decides between its kernel and its reference through one gate, ``primitives._kernels``: CPU tensors,
``global_config.use_native_kernels = False`` and dtypes the kernel does not serve take the reference silently; on a
CUDA device a missing extension (`native_available()` is False) is an error unless ALPA_B200_ALLOW_FALLBACK=1; a
layout the kernel cannot take runs the reference and is recorded in ``primitives.library_fallbacks()``.
"""
import importlib
import os

_native = None
_load_error = None


def _load():
    global _native, _load_error
    if _native is not None or _load_error is not None:
        return _native
    try:
        _native = importlib.import_module("alpa_b200.ops._C")
    except Exception as first:  # noqa: BLE001
        try:
            from alpa_b200.ops import build
            build.build_kernels()
            _native = importlib.import_module("alpa_b200.ops._C")
        except Exception as e:  # noqa: BLE001
            _load_error = (first, e)
            _native = None
    return _native


def native_available() -> bool:
    return _load() is not None


def native_module():
    """The compiled extension; raises if it cannot be loaded."""
    m = _load()
    if m is None:
        raise RuntimeError(f"alpa_b200 native kernels are not available: {_load_error}")
    return m


def allow_fallback() -> bool:
    return os.environ.get("ALPA_B200_ALLOW_FALLBACK", "0") == "1"


from alpa_b200.ops import primitives  # noqa: E402,F401
from alpa_b200.ops.primitives import *  # noqa: E402,F401,F403
