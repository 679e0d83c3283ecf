"""Rank-aware console output and a JSON-lines metrics sink.

The reference only ``print``s: a ``print0`` helper in its benchmark (root rank only,
reference ``benchmarks/bench.py:26-29``), per-batch losses and wall times in the trainers
(``train_two_phase.py:121,150``).  Here the same information goes through one small layer so that
every line is tagged with its rank and every number also lands in a machine-readable file."""
from __future__ import annotations

import json
import logging
import os
import sys
import time
from typing import Any, Dict, Optional

__all__ = ["print0", "get_logger", "MetricsWriter"]


def _rank() -> int:
    from ..parallel.partition import world_rank
    return world_rank()


def print0(*args, P=None, **kwargs) -> None:
    """``print`` on the root only: rank 0 of ``P`` when given, else world rank 0."""
    is_root = (P.rank == 0) if (P is not None and getattr(P, "active", True)) else (P is None and _rank() == 0)
    if is_root:
        print(*args, **kwargs)
        sys.stdout.flush()


class _RankFilter(logging.Filter):
    def filter(self, record):                               # noqa: A003 - logging API
        record.rank = _rank()
        return True


def get_logger(name: str = "dfno_b200", level: Optional[str] = None, all_ranks: bool = False) -> logging.Logger:
    """Logger whose lines read ``[HH:MM:SS r<rank>] message``.  Non-root ranks log warnings and
    above unless ``all_ranks`` (or ``DFNO_LOG_ALL_RANKS=1``); level from ``DFNO_LOG_LEVEL``."""
    log = logging.getLogger(name)
    if not getattr(log, "_dfno_configured", False):
        h = logging.StreamHandler(sys.stdout)
        h.setFormatter(logging.Formatter("[%(asctime)s r%(rank)d] %(message)s", "%H:%M:%S"))
        h.addFilter(_RankFilter())
        log.addHandler(h)
        log.propagate = False
        log._dfno_configured = True
    lvl = (level or os.environ.get("DFNO_LOG_LEVEL", "INFO")).upper()
    everyone = all_ranks or os.environ.get("DFNO_LOG_ALL_RANKS", "0") != "0"
    log.setLevel(lvl if (everyone or _rank() == 0) else "WARNING")
    return log


class MetricsWriter:
    """Append-only JSON-lines file of training / benchmark metrics, one object per ``log`` call:
    ``{"t": unix time, "rank": r, "step": n, ...}``.  One file per rank (``metrics_{rank:04d}.jsonl``)
    unless ``root_only`` -- then only rank 0 writes.  Values that are tensors are converted with
    ``float()`` (a device sync: log losses you already read back)."""

    def __init__(self, out_dir: str, root_only: bool = True, name: str = "metrics"):
        self.rank = _rank()
        self.enabled = (self.rank == 0) or not root_only
        self.path = os.path.join(out_dir, f"{name}_{self.rank:04d}.jsonl")
        self._fh = None
        if self.enabled:
            os.makedirs(out_dir, exist_ok=True)
            self._fh = open(self.path, "a", buffering=1)

    def log(self, step: Optional[int] = None, **values: Any) -> Dict[str, Any]:
        rec: Dict[str, Any] = {"t": round(time.time(), 3), "rank": self.rank}
        if step is not None:
            rec["step"] = int(step)
        for k, v in values.items():
            rec[k] = float(v) if hasattr(v, "item") else v
        if self._fh is not None:
            self._fh.write(json.dumps(rec) + "\n")
        return rec

    def close(self) -> None:
        if self._fh is not None:
            self._fh.close()
            self._fh = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
