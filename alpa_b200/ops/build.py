"""In-tree build of the alpa_b200 native libraries.

Two shared objects are produced next to this file (git-ignored):

* ``_C*.so``       -- sm_90a CUDA kernels + torch bindings  (``alpa_b200/ops/csrc``)
* ``_planner*.so`` -- C++ planner / runtime core (auto-sharding strategy enumeration, cost graph,
                      ILP branch-and-bound, inter-op DP, instruction interpreter)  (``alpa_b200/csrc``)

Kernels are compiled with ``nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo`` (cross-compiles
on a CPU-only box); the binding translation units with g++.  Objects are cached by content hash.
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import subprocess
import sys
import sysconfig
from pathlib import Path

OPS_DIR = Path(__file__).resolve().parent
PKG_DIR = OPS_DIR.parent
KERNEL_SRC = OPS_DIR / "csrc"
PLANNER_SRC = PKG_DIR / "csrc"
BUILD_DIR = PKG_DIR.parent / "build"

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
# NOTE: $CXX may point at a wrapper that links libstdc++ statically, which clashes with
# torch's libstdc++ inside one process; always use the system g++ unless explicitly overridden.
CXX = os.environ.get("ALPA_B200_CXX", "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++")
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "--use_fast_math",
]


def _ext_suffix() -> str:
    return sysconfig.get_config_var("EXT_SUFFIX") or ".so"


def _hash(paths, extra="") -> str:
    h = hashlib.sha256(extra.encode())
    for p in sorted(paths):
        h.update(str(p.name).encode())
        h.update(p.read_bytes())
    return h.hexdigest()[:16]


# ptxas "wgmma pipeline crossing function boundary": a call anywhere in a kernel (printf included) makes ptxas wait
# for every wgmma.mma_async of that kernel to finish before the next one issues.  The build refuses it.
SERIALIZED_WGMMA = "C7510"


def _run(cmd, what, out=None):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(f"[alpa_b200.build] {what} failed:\n{' '.join(map(str, cmd))}\n{r.stdout}\n{r.stderr}\n")
        raise RuntimeError(f"{what} failed")
    if SERIALIZED_WGMMA in r.stdout + r.stderr:
        if out is not None:
            Path(out).unlink(missing_ok=True)  # not cached: the next build reports it again
        sys.stderr.write(f"[alpa_b200.build] {what}: serialized wgmma ({SERIALIZED_WGMMA}):\n"
                         f"{' '.join(map(str, cmd))}\n{r.stdout}\n{r.stderr}\n")
        raise RuntimeError(f"{what}: ptxas serialized wgmma ({SERIALIZED_WGMMA}); remove the call from the kernel")
    return r


def _torch_flags():
    import torch
    from torch.utils import cpp_extension as ce

    inc = [f"-I{p}" for p in ce.include_paths()] + [f"-I{sysconfig.get_paths()['include']}",
                                                    f"-I{CUDA_HOME}/include"]
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    libdir = ce.library_paths()[0]
    return inc, abi, libdir


def _compile_objects(jobs):
    """jobs: list of (cmd, out_path, what). Runs in parallel, skipping existing outputs."""
    todo = [j for j in jobs if not j[1].exists()]
    if not todo:
        return
    with cf.ThreadPoolExecutor(max_workers=min(8, len(todo))) as ex:
        futs = [ex.submit(_run, cmd, what, out) for cmd, out, what in todo]
        for f in futs:
            f.result()


def build_kernels(verbose=False) -> Path:
    """Build alpa_b200/ops/_C.so (CUDA kernels + torch bindings)."""
    out = OPS_DIR / f"_C{_ext_suffix()}"
    cu = sorted(KERNEL_SRC.glob("*.cu"))
    cpp = sorted(KERNEL_SRC.glob("*.cpp"))
    hdr = sorted(list(KERNEL_SRC.glob("*.h")) + list(KERNEL_SRC.glob("*.cuh")))
    tag = _hash(cu + cpp + hdr, " ".join(NVCC_FLAGS))
    stamp = OPS_DIR / "_C.stamp"
    if out.exists() and stamp.exists() and stamp.read_text() == tag:
        return out
    BUILD_DIR.mkdir(exist_ok=True)
    inc, abi, libdir = _torch_flags()
    hdr_tag = _hash(hdr)
    jobs, objs = [], []
    for s in cu:
        o = BUILD_DIR / f"{s.stem}.{_hash([s], hdr_tag + ' '.join(NVCC_FLAGS))}.o"
        objs.append(o)
        jobs.append(([NVCC, *NVCC_FLAGS, f"-I{KERNEL_SRC}", "-c", str(s), "-o", str(o)], o,
                     f"nvcc {s.name}"))
    for s in cpp:
        o = BUILD_DIR / f"{s.stem}.{_hash([s], hdr_tag)}.o"
        objs.append(o)
        jobs.append(([CXX, "-O2", "-std=c++17", "-fPIC", f"-D_GLIBCXX_USE_CXX11_ABI={abi}",
                      "-DTORCH_EXTENSION_NAME=_C", "-DTORCH_API_INCLUDE_EXTENSION_H", *inc,
                      f"-I{KERNEL_SRC}", "-c", str(s), "-o", str(o)], o, f"g++ {s.name}"))
    if verbose:
        print(f"[alpa_b200.build] compiling {sum(1 for j in jobs if not j[1].exists())} kernel objects")
    _compile_objects(jobs)
    _run([CXX, "-shared", "-o", str(out), *map(str, objs), f"-L{libdir}", f"-Wl,-rpath,{libdir}",
          "-ltorch", "-ltorch_cpu", "-ltorch_cuda", "-lc10", "-lc10_cuda", "-ltorch_python",
          f"-L{CUDA_HOME}/lib64", f"-Wl,-rpath,{CUDA_HOME}/lib64", "-lcudart"], "link _C")
    stamp.write_text(tag)
    return out


def build_planner(verbose=False) -> Path:
    """Build alpa_b200/_planner.so (pure C++/pybind11, no torch/CUDA dependency)."""
    out = PKG_DIR / f"_planner{_ext_suffix()}"
    cpp = sorted(PLANNER_SRC.glob("*.cpp"))
    hdr = sorted(PLANNER_SRC.glob("*.h"))
    if not cpp:
        return out
    tag = _hash(cpp + hdr)
    stamp = PKG_DIR / "_planner.stamp"
    if out.exists() and stamp.exists() and stamp.read_text() == tag:
        return out
    BUILD_DIR.mkdir(exist_ok=True)
    import pybind11

    inc = [f"-I{pybind11.get_include()}", f"-I{sysconfig.get_paths()['include']}", f"-I{PLANNER_SRC}"]
    hdr_tag = _hash(hdr)
    jobs, objs = [], []
    for s in cpp:
        o = BUILD_DIR / f"planner_{s.stem}.{_hash([s], hdr_tag)}.o"
        objs.append(o)
        jobs.append(([CXX, "-O2", "-std=c++17", "-fPIC", "-fvisibility=hidden", *inc, "-c", str(s),
                      "-o", str(o)], o, f"g++ {s.name}"))
    if verbose:
        print(f"[alpa_b200.build] compiling {sum(1 for j in jobs if not j[1].exists())} planner objects")
    _compile_objects(jobs)
    _run([CXX, "-shared", "-o", str(out), *map(str, objs), "-ldl"], "link _planner")
    stamp.write_text(tag)
    return out


def build_all(verbose=False):
    return build_planner(verbose), build_kernels(verbose)


if __name__ == "__main__":
    print(build_all(verbose=True))
