import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA GPU (H100); run with -m gpu")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:  # noqa: BLE001
        has_gpu = False
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords and not has_gpu:
            item.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _select_validated_kernels():
    """On a GPU box: check the newest attention forward kernel in a throw-away process before any test touches CUDA and
    pin the previous generation if it misbehaves there (alpa_b200/ops/selfcheck.py) -- one bad kernel must not take the
    whole GPU suite down with it.  The choice is printed in the session header of `-m gpu` runs."""
    try:
        import torch
        on_gpu = torch.cuda.is_available()
    except Exception:  # noqa: BLE001
        on_gpu = False
    if on_gpu:
        from alpa_b200.ops.selfcheck import select_attention_forward
        print(f"[alpa_b200] attention forward kernel for head dim 64: {select_attention_forward()}", flush=True)
    yield


@pytest.fixture
def local_mesh4():
    """An emulated 4-device mesh inside this process (device-free analogue of the reference's
    LocalPhysicalDeviceMesh(jax.local_devices()[:4]))."""
    import alpa_b200 as alpa
    alpa.shutdown()
    alpa.init(cluster="local", num_devices=4)
    yield alpa.get_global_physical_mesh(create_if_not_exist=True)
    alpa.shutdown()
