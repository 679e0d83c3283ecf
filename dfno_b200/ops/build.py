"""In-tree build / load of the sm_90a (Hopper) extension ``dfno_b200._C``.

The shared object is built under ``dfno_b200/_build`` (git-ignored) with
``-gencode arch=compute_90a,code=sm_90a -lineinfo``.  Loading prefers an existing ``.so`` whose
recorded source hash matches; otherwise it (re)builds with ``torch.utils.cpp_extension`` + ninja.
``nvcc`` cross-compiles without a GPU, so ``build()`` is also the CPU-side "does it build" check.
"""
from __future__ import annotations

import hashlib
import importlib.util
import os
import sys
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.normpath(os.path.join(_HERE, "..", "csrc"))
NAME = "dfno_b200_C"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "--extended-lambda", "-Xptxas", "-v",
] + os.environ.get("DFNO_EXTRA_NVCC_FLAGS", "").split()
BUILD_DIR = os.path.normpath(os.path.join(_HERE, "..", "_build"))

_lock = threading.Lock()
_mod = None


def sources():
    out = []
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cpp")):
            out.append(os.path.join(CSRC, f))
    return out


def source_hash() -> str:
    h = hashlib.sha256()
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cpp", ".h", ".cuh")):
            h.update(f.encode())
            with open(os.path.join(CSRC, f), "rb") as fh:
                h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()[:16]


def _so_path() -> str:
    return os.path.join(BUILD_DIR, NAME + ".so")


def _stamp_path() -> str:
    return os.path.join(BUILD_DIR, "source.hash")


def _import_so():
    spec = importlib.util.spec_from_file_location(NAME, _so_path())
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules[NAME] = mod
    return mod


def is_built() -> bool:
    if not (os.path.exists(_so_path()) and os.path.exists(_stamp_path())):
        return False
    with open(_stamp_path()) as f:
        return f.read().strip() == source_hash()


def build(force: bool = False, verbose: bool = False):
    """Compile (if needed) and import the extension."""
    global _mod
    with _lock:
        if _mod is not None and not force:
            return _mod
        import torch  # noqa: F401  (libtorch must be loaded before the extension)
        if force or not is_built():
            from torch.utils.cpp_extension import load
            os.makedirs(BUILD_DIR, exist_ok=True)
            os.environ.setdefault("MAX_JOBS", str(min(8, os.cpu_count() or 4)))
            load(name=NAME, sources=sources(), extra_cuda_cflags=NVCC_FLAGS,
                 extra_cflags=["-O3", "-std=c++17"], extra_include_paths=[CSRC],
                 build_directory=BUILD_DIR, verbose=verbose, with_cuda=True)
            with open(_stamp_path(), "w") as f:
                f.write(source_hash())
            sys.modules.pop(NAME, None)
        _mod = _import_so()
        return _mod


def load():
    """Import the extension, building it first when missing/stale.  Raises on failure: on a
    GPU box the fused ops must never silently fall back."""
    return build(force=False)
