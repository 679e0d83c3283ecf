"""Process/bootstrap helpers: process-group creation from the launcher environment,
device selection (``get_env``), seeding.

Reference: reference ``dfno/utils.py:42-55`` selects CPU / host-staged GPU /
CUDA-aware MPI from ``USE_CUDA`` / ``CUDA_AWARE``.  Here there is one data path per device
type -- gloo for CPU tensors, NCCL + NVLink peer memory for CUDA tensors -- so the two
variables only decide *whether* the GPU is used.
"""
from __future__ import annotations

import os
from contextlib import nullcontext
from datetime import timedelta

import torch
import torch.distributed as dist

__all__ = ["ensure_process_group", "get_env", "seed_all", "local_rank", "shutdown"]


def local_rank() -> int:
    return int(os.environ.get("LOCAL_RANK", os.environ.get("RANK", "0")))


def ensure_process_group(backend: str = None, timeout_s: int = 600) -> bool:
    """Create the default process group from ``RANK``/``WORLD_SIZE`` if a launcher set them.

    Returns True when a (possibly pre-existing) group is active.  One process per GPU:
    the CUDA device is bound to ``LOCAL_RANK`` *before* NCCL initialises.
    """
    if not dist.is_available():
        return False
    if dist.is_initialized():
        return True
    if "RANK" not in os.environ or "WORLD_SIZE" not in os.environ:
        return False
    if int(os.environ["WORLD_SIZE"]) < 1:
        return False
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29500")
    use_cuda = torch.cuda.is_available() and os.environ.get("DFNO_FORCE_CPU", "0") != "1"
    if backend is None:
        backend = "nccl" if use_cuda else "gloo"
    kwargs = {}
    if backend == "nccl":
        dev = torch.device("cuda", local_rank() % torch.cuda.device_count())
        torch.cuda.set_device(dev)
        kwargs["device_id"] = dev
    dist.init_process_group(backend=backend, timeout=timedelta(seconds=timeout_s), **kwargs)
    return True


def shutdown() -> None:
    if dist.is_available() and dist.is_initialized():
        dist.destroy_process_group()


def get_env(P, num_gpus: int = 1):
    """``(use_cuda, cuda_aware, device_ordinal, device, ctx)`` for partition ``P``.

    ``USE_CUDA`` or ``CUDA_AWARE`` in the environment (or an NCCL default group) selects
    the GPU ``rank % num_gpus``; ``ctx`` is a context manager that makes it current.
    """
    cuda_aware = "CUDA_AWARE" in os.environ
    nccl = dist.is_available() and dist.is_initialized() and dist.get_backend() == "nccl"
    use_cuda = ("USE_CUDA" in os.environ or cuda_aware or nccl) and torch.cuda.is_available()
    ordinal = max(P.rank, 0) % max(int(num_gpus), 1)
    if use_cuda:
        if nccl:                       # device was bound at init; keep it
            ordinal = torch.cuda.current_device()
        device = torch.device("cuda", ordinal)
        ctx = torch.cuda.device(device)
    else:
        device = torch.device("cpu")
        ctx = nullcontext()
    return use_cuda, cuda_aware, ordinal, device, ctx


def seed_all(rank: int, base: int = 123) -> None:
    """Per-rank seeding used by the training scripts (``train_two_phase.py:22-23``)."""
    import numpy as np
    torch.manual_seed(rank + base)
    np.random.seed(rank + base)
