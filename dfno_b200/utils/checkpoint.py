"""Checkpoint / resume.

Two formats:

* **per-rank** (the reference's, SURVEY.md §5.4): ``model_{epoch:04d}_{rank:04d}.pt`` /
  ``model_{rank:04d}.pt`` holding ``state_dict()`` of that rank -- root-owned pointwise
  weights are real tensors on rank 0 and zero-volume elsewhere, spectral weights are one
  tensor per non-empty corner of the rank's ``P_y`` slab
  (reference ``training/two_phase/train_two_phase.py:163-169``).  Only loadable on the
  same partition.  This module additionally writes optimizer state, RNG state and
  epoch/step counters next to it so training can *resume* (the reference cannot).
* **global / canonical** (new): one partition-independent dict -- full pointwise weights and,
  per block, the whole truncated spectral weight ``[C, C, 2m_1, .., 2m_{n-1}, m_n]``.  It is
  what :func:`gather_global_state` / :func:`load_global_state` exchange and what lets a
  checkpoint written on one partition (or backend) be loaded on another
  (:func:`reshard_checkpoint`).
"""
from __future__ import annotations

import os
import re
from typing import Any, Dict, Optional

import numpy as np
import torch
import torch.distributed as dist

from ..parallel.decomposition import shard_bounds
from ..parallel.partition import Partition

__all__ = ["gather_global_state", "load_global_state", "save_checkpoint", "load_checkpoint",
           "checkpoint_path", "reshard_checkpoint", "latest_checkpoint",
           "assemble_global_from_files"]


def _unwrap(model):
    """DistributedFNONd wraps the real network lazily."""
    return getattr(model, "net", None) or model


def _is_fused(net) -> bool:
    return hasattr(net, "engine_state_to_global")


# ------------------------------------------------------------------------------------
# global (partition independent) state
# ------------------------------------------------------------------------------------

def gather_global_state(model, to_all: bool = False) -> Optional[Dict[str, torch.Tensor]]:
    """Assemble the canonical state on rank 0 of ``P_x`` (every rank when ``to_all``).

    Collective over ``P_x``.  Tensors are returned on the CPU.
    """
    net = _unwrap(model)
    if _is_fused(net):
        return net.engine_state_to_global(to_all=to_all)
    P_x: Partition = net.P_x
    mine: Dict[str, Any] = {}
    for name, t in net.state_dict().items():
        m = re.match(r"blocks\.(\d+)\.weights\.(\d+)$", name)
        if m:
            blk = net.blocks[int(m.group(1))]
            start, _ = shard_bounds(blk.fft_shape, blk.P_y.shape, blk.P_y.index)
            box = [(sl.start + start[2 + ax], sl.stop + start[2 + ax])
                   for ax, sl in enumerate(blk.slices[int(m.group(2))][2:])]
            mine.setdefault(f"blocks.{m.group(1)}.spectral", []).append((box, t.detach().cpu()))
        elif t.numel() > 0 and (P_x.rank == 0 or not name.startswith(("linear", "blocks"))):
            if P_x.rank == 0:
                mine[name] = t.detach().cpu()
    if P_x.group is None:
        gathered = [mine]
    else:
        gathered = [None] * P_x.size
        dist.all_gather_object(gathered, mine, group=P_x.group)
    if not (to_all or P_x.rank == 0):
        return None
    out: Dict[str, torch.Tensor] = {}
    for part in gathered:
        for k, v in part.items():
            if k.endswith(".spectral"):
                blk = net.blocks[int(k.split(".")[1])]
                if k not in out:
                    out[k] = torch.zeros(blk.width, blk.width, *blk.fft_shape[2:], dtype=blk.dtype_complex)
                for box, piece in v:
                    out[k][(slice(None), slice(None)) + tuple(slice(a, b) for a, b in box)] = piece
            else:
                out[k] = v
    return out


def load_global_state(model, state: Optional[Dict[str, torch.Tensor]], src_is_root_only: bool = False,
                      strict: bool = True) -> None:
    """Load a canonical state into whatever partition/backend ``model`` uses.

    ``state`` must be present on every rank unless ``src_is_root_only`` (then it is
    broadcast from rank 0 of ``P_x`` first)."""
    net = _unwrap(model)
    P_x: Partition = net.P_x
    if src_is_root_only and P_x.group is not None:
        box = [state if P_x.rank == 0 else None]
        dist.broadcast_object_list(box, src=P_x.world_ranks[0], group=P_x.group)
        state = box[0]
    if _is_fused(net):
        net.engine_state_from_global(state, strict=strict)
        return
    own = net.state_dict()
    new: Dict[str, torch.Tensor] = {}
    for name, t in own.items():
        m = re.match(r"blocks\.(\d+)\.weights\.(\d+)$", name)
        if m:
            key = f"blocks.{m.group(1)}.spectral"
            if key not in state:
                if strict:
                    raise KeyError(key)
                continue
            blk = net.blocks[int(m.group(1))]
            start, _ = shard_bounds(blk.fft_shape, blk.P_y.shape, blk.P_y.index)
            sl = blk.slices[int(m.group(2))]
            gsl = (slice(None), slice(None)) + tuple(
                slice(s.start + start[2 + ax], s.stop + start[2 + ax]) for ax, s in enumerate(sl[2:]))
            new[name] = state[key][gsl].to(device=t.device, dtype=t.dtype)
        elif t.numel() == 0:
            new[name] = t
        elif name in state:
            if state[name].numel() != t.numel():          # e.g. a checkpoint of a model with other out_channels
                raise ValueError(f"canonical state entry {name} has shape {list(state[name].shape)}, the model "
                                 f"needs {list(t.shape)}")
            new[name] = state[name].to(device=t.device, dtype=t.dtype).reshape(t.shape)
        elif strict:
            raise KeyError(name)
        else:
            new[name] = t
    if not strict and state and not any(
            (re.match(r"blocks\.(\d+)\.weights\.(\d+)$", n) and f"blocks.{n.split('.')[1]}.spectral" in state) or n in state
            for n in own):
        raise KeyError(f"canonical state matches no parameter of the model (keys: {sorted(state)[:4]}...)")
    net.load_state_dict(new, strict=strict)


# ------------------------------------------------------------------------------------
# per-rank files (reference layout) + training state
# ------------------------------------------------------------------------------------

def checkpoint_path(out_dir: str, rank: int, epoch: Optional[int] = None, kind: str = "model") -> str:
    stem = f"{kind}_{rank:04d}.pt" if epoch is None else f"{kind}_{epoch:04d}_{rank:04d}.pt"
    return os.path.join(out_dir, stem)


def save_checkpoint(model, out_dir: str, epoch: Optional[int] = None, optimizer=None,
                    extra: Optional[Dict[str, Any]] = None, P: Optional[Partition] = None, scheduler=None) -> str:
    """Write this rank's files (with the optimizer's and an lr scheduler's state when given).  Returns the model
    file path."""
    net = _unwrap(model)
    P = P or net.P_x
    if not P.active:                # a world rank outside P_x owns nothing: it must not clobber rank 0's files
        return ""
    rank = P.rank
    os.makedirs(out_dir, exist_ok=True)
    path = checkpoint_path(out_dir, rank, epoch)
    torch.save(net.state_dict(), path)
    extra = dict(extra or {})
    extra.setdefault("plan", "fused" if _is_fused(net) else getattr(net, "plan_kind", extra.get("plan", "reference")))
    train_state = {
        "epoch": epoch,
        "format": "fused-theta" if _is_fused(net) else "portable",
        "engine": net.engine_meta() if _is_fused(net) else None,
        # zeros appended to the lifted field (DistributedFNO(padding=...)); files without the entry are unpadded
        "padding": None if getattr(net, "padding", None) is None else list(net.padding),
        # the grid the *layers* are sharded over (differs from P_x when time/channel workers were folded)
        "partition": tuple(int(s) for s in getattr(net, "P_work", P).shape),
        "world_ranks": P.world_ranks,
        "optimizer": optimizer.state_dict() if optimizer is not None else None,
        "scheduler": scheduler.state_dict() if scheduler is not None else None,
        "rng_cpu": torch.get_rng_state(),
        "rng_cuda": torch.cuda.get_rng_state() if torch.cuda.is_available() else None,
        "rng_numpy": np.random.get_state(),
        "extra": extra,
    }
    torch.save(train_state, checkpoint_path(out_dir, rank, epoch, kind="train"))
    return path


def load_checkpoint(model, out_dir: str, epoch: Optional[int] = None, optimizer=None,
                    restore_rng: bool = True, map_location=None, P: Optional[Partition] = None,
                    scheduler=None) -> Dict[str, Any]:
    """Load this rank's files (same partition as at save time).  Returns the ``extra`` dict
    plus ``epoch``."""
    net = _unwrap(model)
    P = P or net.P_x
    if not P.active:
        return {}
    rank = P.rank
    sd = torch.load(checkpoint_path(out_dir, rank, epoch), map_location=map_location, weights_only=False)
    net.load_state_dict(sd)
    tpath = checkpoint_path(out_dir, rank, epoch, kind="train")
    info: Dict[str, Any] = {"epoch": epoch}
    if os.path.exists(tpath):
        ts = torch.load(tpath, map_location=map_location, weights_only=False)
        if tuple(ts["partition"]) != tuple(int(s) for s in getattr(net, "P_work", P).shape):
            raise ValueError(f"checkpoint was written on partition {ts['partition']}, "
                             f"model uses {tuple(P.shape)}; use reshard_checkpoint()")
        if optimizer is not None and ts["optimizer"] is not None:
            optimizer.load_state_dict(ts["optimizer"])
        if scheduler is not None and ts.get("scheduler") is not None:
            scheduler.load_state_dict(ts["scheduler"])
        if restore_rng:
            torch.set_rng_state(ts["rng_cpu"])
            if ts["rng_cuda"] is not None and torch.cuda.is_available():
                torch.cuda.set_rng_state(ts["rng_cuda"])
            np.random.set_state(ts["rng_numpy"])
        info.update(ts["extra"])
        info["epoch"] = ts["epoch"]
        info["padding"] = ts.get("padding")
    return info


def latest_checkpoint(out_dir: str, rank: int = 0) -> Optional[int]:
    """Largest epoch for which ``model_{epoch}_{rank}.pt`` exists, else None."""
    best = None
    if os.path.isdir(out_dir):
        for f in os.listdir(out_dir):
            m = re.match(rf"model_(\d{{4}})_{rank:04d}\.pt$", f)
            if m:
                best = max(best or -1, int(m.group(1)))
    return best


def assemble_global_from_files(src_dir: str, grid_x, block_in_shape, modes, epoch: Optional[int] = None,
                               plan: str = "reference") -> Dict[str, torch.Tensor]:
    """Rebuild the canonical state from the per-rank files of a run on worker grid
    ``grid_x`` -- pure index arithmetic, no process group needed (so it can run on any
    number of ranks, or offline)."""
    from ..parallel.planner import corner_boxes, make_pencil_plan, spectrum_shape
    from ..parallel.decomposition import index_of_rank
    first = torch.load(checkpoint_path(src_dir, 0, epoch), map_location="cpu", weights_only=False)
    if "theta" in first:            # files of the fused engine: one flat buffer per rank + its segment table
        from ..models.fused import FusedDistributedFNO
        parts, meta = [], None
        for r in range(int(np.prod(grid_x))):
            tpath = checkpoint_path(src_dir, r, epoch, kind="train")
            if not os.path.exists(tpath):
                raise FileNotFoundError(f"{tpath}: fused-engine checkpoints need the train_* file (segment table)")
            meta = torch.load(tpath, map_location="cpu", weights_only=False).get("engine")
            if not meta:
                raise ValueError(f"{tpath} carries no engine segment table; it was written by an older version")
            sd = first if r == 0 else torch.load(checkpoint_path(src_dir, r, epoch), map_location="cpu", weights_only=False)
            parts.append(FusedDistributedFNO.theta_to_canonical(sd["theta"], meta, include_pointwise=r == 0))
        return FusedDistributedFNO.merge_canonical(parts, meta)
    fft_shape = spectrum_shape(block_in_shape, modes)
    pp = make_pencil_plan(grid_x, kind=plan, spectrum=fft_shape)
    n_src = int(np.prod(grid_x))
    n_y = int(np.prod(pp.grid_y))
    out: Dict[str, torch.Tensor] = {}
    for r in range(n_src):
        sd = torch.load(checkpoint_path(src_dir, r, epoch), map_location="cpu", weights_only=False)
        boxes = []
        if r < n_y:
            start, stop = shard_bounds(fft_shape, pp.grid_y, index_of_rank(pp.grid_y, r))
            boxes = [[(a + start[2 + ax], b + start[2 + ax]) for ax, (a, b) in enumerate(box)]
                     for box in corner_boxes(fft_shape, modes, start, stop)]
        for name, t in sd.items():
            m = re.match(r"blocks\.(\d+)\.weights\.(\d+)$", name)
            if m:
                key = f"blocks.{m.group(1)}.spectral"
                if key not in out:
                    out[key] = torch.zeros(t.shape[0], t.shape[1], *fft_shape[2:], dtype=t.dtype)
                box = boxes[int(m.group(2))]
                out[key][(slice(None), slice(None)) + tuple(slice(a, b) for a, b in box)] = t
            elif t.numel() > 0 and (r == 0 or name not in out):
                out[name] = t
    return out


def reshard_checkpoint(src_dir: str, dst_model, epoch: Optional[int] = None, src_grid=None,
                       src_plan: Optional[str] = None) -> None:
    """Load per-rank files written on *another* partition into ``dst_model`` (same
    architecture).  Every destination rank reads the source files, rebuilds the canonical
    state and slices its own shard."""
    net = _unwrap(dst_model)
    tpath = checkpoint_path(src_dir, 0, epoch, kind="train")
    meta = torch.load(tpath, weights_only=False) if os.path.exists(tpath) else {}
    grid = tuple(src_grid) if src_grid is not None else tuple(meta["partition"])
    plan = src_plan or meta.get("extra", {}).get("plan", "reference")
    if plan == "fused":
        plan = "reference"          # irrelevant for theta files (assemble_global_from_files reads the segment table)
    state = assemble_global_from_files(src_dir, grid, net.block_in_shape, net.modes, epoch, plan)
    load_global_state(dst_model, state, strict=False)
