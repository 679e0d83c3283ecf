"""Timing helpers.

``CommTimer`` reproduces the reference's per-module ``dt_comm`` accounting
(reference ``dfno/dfno.py:54-60,242-289``) but can be told to synchronise the device so
the number means something on an asynchronous GPU stream.  ``cuda_time_ms`` is the
benchmark-grade device timer (CUDA events, explicit synchronisation on both sides).
"""
from __future__ import annotations

import os
import time
from contextlib import contextmanager

import torch

__all__ = ["CommTimer", "cuda_time_ms", "nvtx_range"]

_SYNC = os.environ.get("DFNO_SYNC_TIMERS", "0") == "1"


class CommTimer:
    def __init__(self):
        self.seconds = 0.0
        self._t0 = 0.0

    def reset(self) -> None:
        self.seconds = 0.0

    def __enter__(self):
        if _SYNC and torch.cuda.is_available():
            torch.cuda.synchronize()
        self._t0 = time.perf_counter()
        return self

    def __exit__(self, *exc):
        if _SYNC and torch.cuda.is_available():
            torch.cuda.synchronize()
        self.seconds += time.perf_counter() - self._t0
        return False


def cuda_time_ms(fn, iters: int = 10, warmup: int = 3, flush_l2: bool = True):
    """Median/mean/min device time of ``fn()`` in ms (CUDA events on the current stream)."""
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.int8, device="cuda") if flush_l2 else None
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
    times.sort()
    return {"median": times[len(times) // 2], "min": times[0], "mean": sum(times) / len(times)}


@contextmanager
def nvtx_range(name: str):
    """NVTX range when CUDA is present (the reference installs ``nvtx`` but never uses it)."""
    on = torch.cuda.is_available()
    if on:
        torch.cuda.nvtx.range_push(name)
    try:
        yield
    finally:
        if on:
            torch.cuda.nvtx.range_pop()
