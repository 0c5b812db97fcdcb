"""First hardware runs of code written after this round's GPU budget was spent (runs last).  Each check runs in a
throw-away process with a timeout, so a wrong barrier protocol cannot hang the session, and is marked
xfail(strict=False): the suite reports XPASS when the new path works on the H100 and XFAIL -- not a red suite -- when
it does not; nothing on a default execution path depends on these kernels (both are opt-in)."""
import os
import subprocess
import sys
import warnings

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


_BUDGET_S = 780.0          # all checks of this file together: the GPU suite must stay well inside the driver's step limit
_spent = [0.0]


def _run(script, timeout, *args):
    import time
    left = _BUDGET_S - _spent[0]
    if left < 30:
        pytest.skip("time budget of the first-hardware-run checks is used up")
    timeout = min(timeout, left)
    t0 = time.time()
    try:
        return _run_inner(script, timeout, *args)
    finally:
        _spent[0] += time.time() - t0


def _run_inner(script, timeout, *args):
    env = dict(os.environ, ALPA_B200_REQUIRE_NATIVE="1",
               PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", script), *args], capture_output=True, text=True,
                       timeout=timeout, env=env, cwd=ROOT)
    print(r.stdout[-4000:])
    print(r.stderr[-2000:])
    # the result lines go to pytest's warnings summary: it is printed even for xpassed / xfailed tests under -q, so the
    # numbers of the first hardware run end up in the session log either way
    keep = [ln.strip() for ln in r.stdout.splitlines() if ln.startswith(("native comm", "p2p", "cached pipeshard", "attention_cached", "train feature", "pack ", "BENCH "))]
    if r.returncode != 0:
        keep += ["rc=%d" % r.returncode] + [ln.strip() for ln in r.stderr.splitlines()[-6:]]
    warnings.warn("first hardware run of %s: %s" % (script, " | ".join(keep)[-1800:]))
    return r


@pytest.mark.xfail(strict=False, reason="native communication module (dlopen'ed NCCL / CUDA runtime): first hardware run")
def test_native_comm_module_first_hardware_run():
    r = _run("gpu_check_native_comm_1gpu.py", 120)
    assert r.returncode == 0 and "native comm 1-gpu check: ok" in r.stdout


@pytest.mark.xfail(strict=False, reason="ops.attention_cached on the native prefill / decode-attention kernels: first hardware run")
def test_attention_cached_primitive_first_hardware_run():
    r = _run("gpu_check_attention_cached.py", 120)
    assert r.returncode == 0 and "attention_cached check: ok" in r.stdout


@pytest.mark.xfail(strict=False, reason="KV-cached decoder through @parallelize on a GPU (attention_cached on the native kernels): first hardware run")
def test_cached_pipeshard_decoder_first_hardware_run():
    r = _run("gpu_check_cached_pipeshard.py", 300)
    assert r.returncode == 0 and "cached pipeshard check: ok" in r.stdout


@pytest.mark.xfail(strict=False, reason="gradient accumulation and rematerialisation executables on the native kernels: first hardware run")
def test_grad_accumulation_and_remat_first_hardware_run():
    r = _run("gpu_check_train_features.py", 240)
    assert r.returncode == 0 and "train feature check: ok" in r.stdout


@pytest.mark.xfail(strict=False, reason="resharding pack / unpack kernel (pack_sm90.cu): first hardware run")
def test_resharding_pack_kernel_first_hardware_run():
    r = _run("gpu_check_pack.py", 120)
    assert r.returncode == 0 and "pack check: ok" in r.stdout


@pytest.mark.xfail(strict=False, reason="informational: GEMM / attention timings of the kernels at HEAD on this box")
def test_kernel_timings_at_head():
    """Not a validation (the numerics of these kernels are checked by tests/test_gemm_numerics.py and
    tests/test_kernel_numerics.py): runs the timing sections of scripts/gpu_check.py so that the session log carries
    TFLOPS of the wgmma GEMM (against cuBLAS) and of the attention forward / backward as built from this commit."""
    r = _run("gpu_check.py", 240, "gemm_bench", "attn")
    assert r.returncode == 0
