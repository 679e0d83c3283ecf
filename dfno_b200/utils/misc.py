"""Small utilities of the public namespace (reference ``dfno/utils.py``)."""
from __future__ import annotations

import subprocess
import time
from typing import Any, Dict, Sequence

import numpy as np
import torch

from ..parallel.decomposition import (assemble_slices, compute_subtensor_shapes_balanced,
                                      compute_subtensor_start_indices,
                                      compute_subtensor_stop_indices)

__all__ = ["compute_distribution_info", "alphabet", "unit_guassian_normalize",
           "unit_gaussian_normalize", "unit_gaussian_denormalize", "get_gpu_memory",
           "profile_gpu_memory", "TensorStructure"]


class TensorStructure:
    """Shape/dtype carrier (DistDL utility the reference imports; SURVEY.md §2.2 E8)."""

    def __init__(self, tensor=None):
        self.shape = None if tensor is None else tuple(tensor.shape)
        self.dtype = None if tensor is None else tensor.dtype
        self.requires_grad = False if tensor is None else tensor.requires_grad


def compute_distribution_info(P, shape: Sequence[int]) -> Dict[str, Any]:
    """Balanced-decomposition tables of a global ``shape`` over partition ``P``.

    Keys: ``shapes``/``starts``/``stops`` (arrays over the whole grid) and, for an active
    rank, ``index``/``shape``/``start``/``stop``/``slice`` (``utils.py:58-70``)."""
    shapes = compute_subtensor_shapes_balanced(shape, P.shape)
    info = {"shapes": shapes,
            "starts": compute_subtensor_start_indices(shapes),
            "stops": compute_subtensor_stop_indices(shapes)}
    if P.active:
        idx = tuple(P.index)
        info.update(index=idx, shape=info["shapes"][idx], start=info["starts"][idx],
                    stop=info["stops"][idx])
        info["slice"] = assemble_slices(info["start"], info["stop"])
    else:
        info.update(index=None, shape=None, start=None, stop=None, slice=None)
    return info


def alphabet(n: int, as_array: bool = False):
    letters = [chr(ord("a") + i) for i in range(n)]
    return letters if as_array else "".join(letters)


def unit_gaussian_normalize(x: torch.Tensor, eps: float = 1e-6):
    """Standardise over dim 0; returns ``(x_hat, mu, std)``."""
    mu = x.mean(dim=0, keepdim=True)
    std = x.std(dim=0, keepdim=True)
    return (x - mu) / (std + eps), mu, std


#: the reference's (misspelt) public name, kept so scripts run unchanged (``utils.py:90``)
unit_guassian_normalize = unit_gaussian_normalize


def unit_gaussian_denormalize(x: torch.Tensor, mu: torch.Tensor, std: torch.Tensor, eps: float = 1e-6):
    return x * (std + eps) + mu


def get_gpu_memory():
    """Used memory (MiB) of every visible GPU, from ``nvidia-smi``."""
    try:
        out = subprocess.check_output(
            ["nvidia-smi", "--query-gpu=memory.used", "--format=csv,noheader,nounits"],
            stderr=subprocess.STDOUT)
    except (OSError, subprocess.CalledProcessError) as e:
        raise RuntimeError(f"nvidia-smi query failed: {e}") from e
    return [int(tok) for tok in out.decode().split()]


def profile_gpu_memory(outfile, dt: float = 1.0, max_samples: int = None):
    """Poll :func:`get_gpu_memory` every ``dt`` seconds into a CSV (meant for a daemon
    process, reference ``benchmarks/bench.py:57-62``)."""
    t0 = time.time()
    n = 0
    with open(outfile, "w") as f:
        while max_samples is None or n < max_samples:
            row = [f"{time.time() - t0:.3f}"] + [str(m) for m in get_gpu_memory()]
            f.write(", ".join(row) + "\n")
            f.flush()
            n += 1
            time.sleep(dt)
