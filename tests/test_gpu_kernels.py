"""GPU smoke checks: the native extension is loaded, and one small training step through the public API lowers the
loss.  The kernels themselves are checked against float64 references in the *_numerics.py tests."""
import pytest

pytestmark = pytest.mark.gpu


def test_native_extension_loaded():
    from alpa_b200 import ops
    assert ops.native_available(), "sm_90a extension must be built in-tree (python -m alpa_b200.ops.build)"
    assert hasattr(ops.native_module(), "gemm")


def test_train_step_decreases_loss():
    import __graft_entry__ as g
    g.smoke()
