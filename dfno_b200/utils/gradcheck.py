"""Taylor-remainder gradient check for (distributed) modules.

For every parameter ``p`` with a random direction ``dp`` the zeroth-order remainder
``|J(p+h dp) - J(p)|`` must decay like ``h`` and the first-order remainder
``|J(p+h dp) - J(p) - h <grad J, dp>|`` like ``h^2``; slopes are fitted in log-log space.
Same idea as reference ``tests/gradient_test.py:40-132``, with the distributed
details done properly:

* the objective is the **global** ``1/2 ||f(x) - y0||^2`` (local terms all-reduced), not a
  per-rank norm;
* the directional derivative ``<grad, dp>`` is all-reduced too, so parameters that are
  sharded (spectral weights) or root-owned (pointwise weights) are handled uniformly and
  no ad-hoc rescaling of the fit is needed;
* perturbations are applied on the owning rank(s) only; every rank evaluates the same
  number of forwards, so collectives stay matched.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn

__all__ = ["GradientTestResult", "gradient_test"]


@dataclass
class GradientTestResult:
    name: str
    active: bool
    converged: Tuple[bool, bool]
    convergence: Tuple[List[float], List[float]]
    steps: List[float]
    slopes: Tuple[float, float] = (float("nan"), float("nan"))

    @property
    def ok(self) -> bool:
        return (not self.active) or (self.converged[0] and self.converged[1])

    def __str__(self) -> str:
        e0 = ", ".join(f"{v:.2e}" for v in self.convergence[0])
        e1 = ", ".join(f"{v:.2e}" for v in self.convergence[1])
        return (f"==== {self.name} ====\nactive: {self.active}\n"
                f"O(h) slope {self.slopes[0]:.3f} ok={self.converged[0]}  err=[{e0}]\n"
                f"O(h^2) slope {self.slopes[1]:.3f} ok={self.converged[1]}  err=[{e1}]")


def _allsum(v: float, group) -> float:
    if group is None:
        return float(v)
    t = torch.tensor([float(v)], dtype=torch.float64)
    dist.all_reduce(t, group=group)
    return float(t.item())


def gradient_test(f: nn.Module, input_shape: Sequence[int], max_iter: int = 8,
                  dtype: torch.dtype = torch.float64, group="auto", h0: float = 1.0,
                  rtol: float = 0.1, names: Optional[Sequence[str]] = None,
                  seed: int = 0) -> Iterator[GradientTestResult]:
    """Yield one :class:`GradientTestResult` per named parameter of ``f``.

    ``input_shape`` is this rank's *local* input shape.  ``group`` is the process group the
    objective is summed over (default: ``f.P_x.group`` when present)."""
    if group == "auto":
        P = getattr(f, "P_x", None)
        group = P.group if (P is not None and P.active) else None
    rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else 0
    gen = torch.Generator().manual_seed(1234 + seed + 7919 * rank)
    x0 = 1 + torch.rand(*input_shape, dtype=dtype, generator=gen)
    x1 = 1 + torch.rand(*input_shape, dtype=dtype, generator=gen)
    with torch.no_grad():
        y0 = f(x0).detach()

    def objective() -> torch.Tensor:
        return 0.5 * (f(x1) - y0).pow(2).sum()

    # Ranks own different parameter sets (spectral shards exist only where modes live), so
    # agree on the union of names first: every rank must run every trial.
    local = dict(f.named_parameters())
    all_names = list(local)
    if group is not None:
        gathered = [None] * dist.get_world_size(group)
        dist.all_gather_object(gathered, all_names, group=group)
        all_names = list(dict.fromkeys(n for lst in gathered for n in lst))

    for name in all_names:
        if names is not None and name not in names:
            continue
        p = local.get(name)
        owns = p is not None and p.numel() > 0 and p.requires_grad
        saved = p.data.clone() if p is not None else None
        if owns:
            rdt = p.real.dtype if p.is_complex() else p.dtype
            def rnd():
                r = torch.rand(*p.shape, dtype=rdt, generator=gen)
                if p.is_complex():
                    r = torch.complex(r, torch.rand(*p.shape, dtype=rdt, generator=gen))
                return r
            p0 = (saved + 0.1 * rnd() * saved.abs().mean().clamp_min(1e-3)).to(p.dtype)
            dp = (1e-1 * (0.5 + rnd()) * saved.abs().mean().clamp_min(1e-3)).to(p.dtype)
            p.data = p0.clone()
        f.zero_grad(set_to_none=True)
        J0 = objective()
        J0.backward()
        gdx_local = 0.0
        if owns and p.grad is not None:
            # real inner product; for complex parameters torch's grad convention gives
            # dJ = Re <grad, dp>
            gdx_local = float(torch.sum((p.grad.conj() * dp).real if p.is_complex() else p.grad * dp))
        gdx = _allsum(gdx_local, group)
        J0v = _allsum(float(J0.detach()), group)
        active = bool(_allsum(1.0 if owns else 0.0, group) > 0)

        hs, e0, e1 = [], [], []
        h = h0
        for _ in range(max_iter):
            if owns:
                p.data = p0 + h * dp
            with torch.no_grad():
                Jh = _allsum(float(objective()), group)
            hs.append(h)
            e0.append(abs(Jh - J0v))
            e1.append(abs(Jh - J0v - h * gdx))
            h *= 0.5
        if p is not None:
            p.data = saved
        f.zero_grad(set_to_none=True)

        slopes = (float("nan"), float("nan"))
        conv = (False, False)
        if active:
            tiny = 1e-13 * max(abs(J0v), 1.0)
            keep = [i for i in range(len(hs)) if e1[i] > tiny and e0[i] > tiny]
            if len(keep) >= 3:
                lh = np.log10([hs[i] for i in keep])
                tail = keep[len(keep) // 2:]      # small-h regime: first- and second-order terms
                                                  # can cancel at large h
                s0 = float(np.polyfit(np.log10([hs[i] for i in tail]),
                                      np.log10([e0[i] for i in tail]), 1)[0])
                s1 = float(np.polyfit(lh, np.log10([e1[i] for i in keep]), 1)[0])
                slopes = (s0, s1)
                # zeroth-order remainder: decays (at least) linearly -- it looks quadratic when
                # the directional derivative is small against the curvature term at these h
                conv = (bool(1.0 - rtol <= s0 <= 2.0 + 2 * rtol), bool(np.isclose(s1, 2.0, rtol=rtol)))
            else:
                # remainder already at round-off: the function is (numerically) affine in p
                conv, slopes = (True, True), (1.0, 2.0)
        yield GradientTestResult(name, active, conv, (e0, e1), hs, slopes)
