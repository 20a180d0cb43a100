"""Build / load the sm_90a CUDA extension (in-tree, so the .so travels with the repo).

All kernels live in ``csrc/`` and are compiled with
``-gencode arch=compute_90a,code=sm_90a -lineinfo`` into ``poseidon_b200/_ext/poseidon_b200_C.so``;
ops register themselves under ``torch.ops.poseidon``.
"""
from __future__ import annotations

import glob
import os
import threading

import torch

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
CSRC = os.path.join(_ROOT, "csrc")
EXT_DIR = os.path.join(_ROOT, "poseidon_b200", "_ext")
EXT_NAME = "poseidon_b200_C"
_lock = threading.Lock()
_loaded = False

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "-Xptxas", "-v", "--threads", "4",
    "-DPSD_SPIN_LIMIT=67108864u",
]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "**", "*.cu"), recursive=True) +
                  glob.glob(os.path.join(CSRC, "**", "*.cpp"), recursive=True))


def so_path() -> str:
    return os.path.join(EXT_DIR, EXT_NAME + ".so")


def _stale() -> bool:
    so = so_path()
    if not os.path.exists(so):
        return True
    t = os.path.getmtime(so)
    deps = sources() + glob.glob(os.path.join(CSRC, "**", "*.cuh"), recursive=True) + \
        glob.glob(os.path.join(CSRC, "**", "*.h"), recursive=True)
    return any(os.path.getmtime(f) > t for f in deps)


def build_extension(verbose: bool = False, force: bool = False) -> str:
    """Compile (if stale) and return the .so path.  Works without a GPU (nvcc cross-compiles)."""
    from torch.utils import cpp_extension
    os.makedirs(EXT_DIR, exist_ok=True)
    if force or _stale():
        os.environ.setdefault("MAX_JOBS", str(max(2, (os.cpu_count() or 4))))
        cpp_extension.load(
            name=EXT_NAME, sources=sources(), extra_cflags=["-O3", "-std=c++17"],
            extra_cuda_cflags=NVCC_FLAGS, extra_include_paths=[CSRC, os.path.join(CSRC, "gemm")],
            build_directory=EXT_DIR, verbose=verbose,
            is_python_module=False, with_cuda=True)
    return so_path()


def load_extension(build_if_missing: bool = True) -> bool:
    """Load the ops into ``torch.ops.poseidon``.  Raises if the extension cannot be had on a CUDA
    box (the sm100 engine never silently falls back to library kernels)."""
    global _loaded
    with _lock:
        if _loaded:
            return True
        so = so_path()
        if not os.path.exists(so):
            if not build_if_missing:
                raise RuntimeError(f"{so} not built; run `python -c 'import __graft_entry__ as g; g.build()'`")
            build_extension()
        torch.ops.load_library(so)
        _loaded = True
        return True


def is_loaded() -> bool:
    return _loaded
