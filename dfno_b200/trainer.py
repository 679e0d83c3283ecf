"""Training-step driver: host batch -> device (pinned, asynchronous, double buffered) ->
forward -> distributed loss -> backward -> optimizer, loss read back to the host.

This is the loop of reference ``training/two_phase/train_two_phase.py:99-121`` as a
reusable object.  The H2D copies of step ``i+1`` run on a side stream while step ``i``
computes; the loss value is read back from a pinned scalar.
"""
from __future__ import annotations

from typing import Callable, Optional, Tuple

import torch

__all__ = ["Trainer", "InferenceSession"]


class Trainer:
    def __init__(self, model, criterion, optimizer, device: Optional[torch.device] = None,
                 target_dtype: Optional[torch.dtype] = None, cuda_graph: bool = False,
                 before_step: Optional[Callable[[], None]] = None):
        """``before_step``: called between the backward and ``optimizer.step()``, e.g. gradient clipping for a
        ``torch.optim`` optimizer (:class:`FusedAdam` clips inside its step: ``max_grad_norm``)."""
        self.model, self.criterion, self.optimizer = model, criterion, optimizer
        self.before_step = before_step
        self.device = torch.device(device) if device is not None else next(model.parameters()).device
        self.cuda = self.device.type == "cuda"
        self.copy_stream = torch.cuda.Stream(device=self.device) if self.cuda else None
        self._slots = [None, None]
        self._ready = [None, None]
        self._next = 0
        self._pending = None
        self.target_dtype = target_dtype
        self._loss_host = torch.zeros((), dtype=torch.float32).pin_memory() if self.cuda else torch.zeros(())
        self.h2d_bytes = 0
        self.d2h_bytes = 0
        # CUDA-graph replay of the whole step (forward, loss, backward, optimizer): one launch per
        # step instead of a few hundred.  Falls back to eager execution if capture is not possible.
        self.cuda_graph = bool(cuda_graph) and self.cuda
        self._graph = None
        self._graph_key = None
        self._graph_failed = False
        self.graph_kernel_launches = 0

    # -------------------------------------------------------------------- data movement
    def _upload(self, x_host: torch.Tensor, y_host: torch.Tensor):
        if not self.cuda:
            return x_host, y_host, None
        slot = self._next
        self._next ^= 1
        if self._slots[slot] is None or self._slots[slot][0].shape != x_host.shape \
                or self._slots[slot][1].shape != y_host.shape:
            self._slots[slot] = (torch.empty_like(x_host, device=self.device),
                                 torch.empty_like(y_host, device=self.device))
        xd, yd = self._slots[slot]
        cur = torch.cuda.current_stream(self.device)
        self.copy_stream.wait_stream(cur)          # the slot's previous consumer has been enqueued
        with torch.cuda.stream(self.copy_stream):
            xd.copy_(x_host, non_blocking=True)
            yd.copy_(y_host, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.copy_stream)
        self.h2d_bytes = x_host.numel() * x_host.element_size() + y_host.numel() * y_host.element_size()
        return xd, yd, ev

    def prefetch(self, x_host: torch.Tensor, y_host: torch.Tensor) -> None:
        """Start copying the *next* batch while the current step runs."""
        self._pending = self._upload(x_host, y_host)

    # -------------------------------------------------------------------- one step
    def step(self, x_host: torch.Tensor, y_host: torch.Tensor,
             next_batch: Optional[Tuple[torch.Tensor, torch.Tensor]] = None) -> float:
        """One optimisation step on a host batch (this rank's shard).  Returns the loss
        (valid on the root rank, 0 elsewhere -- the distributed-loss convention)."""
        if self._pending is not None:
            xd, yd, ev = self._pending
            self._pending = None
        else:
            xd, yd, ev = self._upload(x_host, y_host)
        if ev is not None:
            torch.cuda.current_stream(self.device).wait_event(ev)
        if next_batch is not None:
            self.prefetch(*next_batch)
        loss = self._graphed(xd, yd) if (self.cuda_graph and not self._graph_failed) else self._eager(xd, yd)
        if self.cuda:
            self._loss_host.copy_(loss.detach(), non_blocking=True)
            torch.cuda.current_stream(self.device).synchronize()
            self.d2h_bytes = 4
            return float(self._loss_host)
        self.d2h_bytes = 0
        return float(loss.detach())

    def step_on_device(self, xd: torch.Tensor, yd: torch.Tensor) -> torch.Tensor:
        """One optimisation step on a batch that already lives on the device; returns the loss
        as a device tensor (no host synchronisation).  Replays the captured graph when enabled."""
        return self._graphed(xd, yd) if (self.cuda_graph and not self._graph_failed) else self._eager(xd, yd)

    def _eager(self, xd: torch.Tensor, yd: torch.Tensor) -> torch.Tensor:
        self.optimizer.zero_grad(set_to_none=True)
        y_hat = self.model(xd)
        loss = self.criterion(y_hat, yd)
        loss.backward()
        if self.before_step is not None:
            self.before_step()
        self.optimizer.step()
        return loss

    def _graphed(self, xd: torch.Tensor, yd: torch.Tensor) -> torch.Tensor:
        opt = self.optimizer
        key = opt.graph_key() if hasattr(opt, "graph_key") else None
        if self._graph is not None and key != self._graph_key:
            # the captured step baked in other hyperparameters: capture again, on the device-hyperparameter path so
            # that later changes need no further capture
            if key[0] == "host" and hasattr(opt, "use_device_hparams"):
                opt.use_device_hparams()
                key = opt.graph_key()
            self._graph = None
        if self._graph is None:
            try:
                self._gx, self._gy = torch.empty_like(xd), torch.empty_like(yd)
                self._gx.copy_(xd); self._gy.copy_(yd)
                # the warm-up steps and the capture pass must not train: snapshot parameters / optimizer state and
                # put them back afterwards (in place -- the captured graph holds these very tensors), so the first
                # batch gets exactly one update and host / device step counters agree
                snap = self._snapshot_training_state()
                side = torch.cuda.Stream(device=self.device)
                side.wait_stream(torch.cuda.current_stream(self.device))
                with torch.cuda.stream(side):                 # warm-up off the capturing stream
                    for _ in range(2):
                        self._eager(self._gx, self._gy)
                torch.cuda.current_stream(self.device).wait_stream(side)
                torch.cuda.synchronize(self.device)
                counter = getattr(self.model, "_C", None)
                c0 = getattr(counter, "count", 0)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    self._gloss = self._eager(self._gx, self._gy).detach()
                self.graph_kernel_launches = getattr(counter, "count", 0) - c0
                self._restore_training_state(snap)
                self._graph, self._graph_key = graph, key
                self._graph_steps_py = getattr(self.optimizer, "step_count", None)
            except Exception as e:                            # noqa: BLE001 - capture is an optimisation
                import warnings
                warnings.warn(f"CUDA-graph capture of the training step failed ({type(e).__name__}: {e}); "
                              f"running eagerly")
                self._graph_failed = True
                torch.cuda.synchronize(self.device)
                return self._eager(xd, yd)
        self._gx.copy_(xd, non_blocking=True)
        self._gy.copy_(yd, non_blocking=True)
        if hasattr(opt, "before_replay"):
            opt.before_replay()                               # this replay's lr, betas, ... into the device scalars
        self._graph.replay()
        if hasattr(opt, "step_count"):
            opt.step_count += 1                               # host mirror of the device-side counter
        # what the step wrapper of an attached lr scheduler records on an eager step (else scheduler.step() warns
        # that it ran before optimizer.step())
        opt._opt_called = True
        counter = getattr(self.model, "_C", None)
        if hasattr(counter, "count"):
            counter.count += self.graph_kernel_launches
        return self._gloss

    # -------------------------------------------------------------------- state snapshot around graph capture
    @torch.no_grad()
    def _snapshot_training_state(self):
        opt = self.optimizer
        snap = {"params": [(p, p.detach().clone()) for p in self.model.parameters()], "tensors": [], "attrs": {}}
        if hasattr(opt, "m") and hasattr(opt, "v"):                      # FusedAdam: flat moment buffers + counters
            for name in ("m", "v", "step_dev"):
                t = getattr(opt, name, None)
                if torch.is_tensor(t):
                    snap["tensors"].append((t, t.clone()))
            snap["attrs"]["step_count"] = getattr(opt, "step_count", 0)
        elif hasattr(opt, "state"):                                      # torch.optim.*: per-parameter state dicts
            snap["had_state"] = {id(p) for p in opt.state}
            for st in opt.state.values():
                for k, v in st.items():
                    if torch.is_tensor(v):
                        snap["tensors"].append((v, v.clone()))
        return snap

    @torch.no_grad()
    def _restore_training_state(self, snap) -> None:
        for p, v in snap["params"]:
            p.data.copy_(v)
        for t, v in snap["tensors"]:
            t.copy_(v)
        opt = self.optimizer
        for k, v in snap["attrs"].items():
            setattr(opt, k, v)
        if "had_state" in snap:               # state created during the warm-up: zero it (lazy init happened there)
            for p, st in opt.state.items():
                if id(p) not in snap["had_state"]:
                    for k, v in st.items():
                        if torch.is_tensor(v):
                            v.zero_()
        torch.cuda.synchronize(self.device)

    @torch.no_grad()
    def evaluate(self, x_host: torch.Tensor, y_host: torch.Tensor) -> float:
        xd, yd, ev = self._upload(x_host, y_host)
        if ev is not None:
            torch.cuda.current_stream(self.device).wait_event(ev)
        return float(self.criterion(self.model(xd), yd))



class InferenceSession:
    """Forward-only serving loop: pinned host shard in -> (CUDA-graph replayed) forward -> pinned host
    shard out.  The counterpart of :class:`Trainer` for deployment; the reference only has the one-shot
    script reference ``training/two_phase/test_two_phase.py``.

    ``run`` is synchronous (returns when the output is on the host); ``submit`` / ``result`` split it so
    that the upload of request ``i+1`` overlaps the forward of request ``i``.  With ``cuda_graph`` the
    forward of a fixed input shape is captured once and replayed; capture failures fall back to eager
    launches, as in :class:`Trainer`."""

    def __init__(self, model, device: Optional[torch.device] = None, cuda_graph: bool = True):
        self.model = model
        self.device = torch.device(device) if device is not None else next(model.parameters()).device
        self.cuda = self.device.type == "cuda"
        self.cuda_graph = bool(cuda_graph) and self.cuda
        self.copy_stream = torch.cuda.Stream(device=self.device) if self.cuda else None
        self._graph = None
        self._graph_failed = False
        self._gx = self._gy = None
        self._out_host = None
        self._inflight = None
        self.requests = 0
        model.eval()

    @torch.no_grad()
    def _forward(self, xd: torch.Tensor) -> torch.Tensor:
        if not self.cuda_graph or self._graph_failed:
            return self.model(xd)
        if self._graph is None or self._gx.shape != xd.shape or self._gx.dtype != xd.dtype:
            try:
                self._gx = torch.empty_like(xd)
                self._gx.copy_(xd)
                side = torch.cuda.Stream(device=self.device)
                side.wait_stream(torch.cuda.current_stream(self.device))
                with torch.cuda.stream(side):                 # warm-up (allocations, lazy plans) off-capture
                    for _ in range(2):
                        self.model(self._gx)
                torch.cuda.current_stream(self.device).wait_stream(side)
                torch.cuda.synchronize(self.device)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    self._gy = self.model(self._gx)
                self._graph = graph
            except Exception as e:                            # noqa: BLE001 - capture is an optimisation
                import warnings
                warnings.warn(f"CUDA-graph capture of the forward failed ({type(e).__name__}: {e}); running eagerly")
                self._graph_failed, self._graph = True, None
                torch.cuda.synchronize(self.device)
                return self.model(xd)
        self._gx.copy_(xd, non_blocking=True)
        self._graph.replay()
        return self._gy

    def submit(self, x_host: torch.Tensor) -> None:
        """Enqueue one request: async H2D on the copy stream, forward, async D2H into a pinned buffer."""
        if self._inflight is not None:
            raise RuntimeError("collect the previous result() first (one request in flight)")
        if not self.cuda:
            with torch.no_grad():
                self._inflight = (self.model(x_host), None)
            return
        cur = torch.cuda.current_stream(self.device)
        self.copy_stream.wait_stream(cur)
        with torch.cuda.stream(self.copy_stream):
            xd = x_host.to(self.device, non_blocking=True)
            up = torch.cuda.Event()
            up.record(self.copy_stream)
        cur.wait_event(up)
        xd.record_stream(cur)
        y = self._forward(xd)
        if self._out_host is None or self._out_host.shape != y.shape or self._out_host.dtype != y.dtype:
            self._out_host = torch.empty(y.shape, dtype=y.dtype).pin_memory()
        self._out_host.copy_(y, non_blocking=True)
        done = torch.cuda.Event()
        done.record(cur)
        self._inflight = (self._out_host, done)

    def result(self) -> torch.Tensor:
        """Block until the submitted request is on the host; returns this rank's output shard (a pinned
        buffer that the next request overwrites -- clone it to keep it)."""
        if self._inflight is None:
            raise RuntimeError("nothing submitted")
        out, done = self._inflight
        self._inflight = None
        if done is not None:
            done.synchronize()
        self.requests += 1
        return out

    def run(self, x_host: torch.Tensor) -> torch.Tensor:
        self.submit(x_host)
        return self.result()
