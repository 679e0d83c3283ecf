import torch
import torch.distributed as dist

from ..backend.backend import _on


class DistributedBatchNorm(torch.nn.Module):
    """Per-channel batch norm with statistics summed over all workers.  The reference only constructs it
    (reference ``dfno/dfno.py:325-326``; it is commented out of the forward)."""

    def __init__(self, P_x, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True,
                 device=None, dtype=None):
        super().__init__()
        self.P_x, self.eps, self.momentum = P_x, eps, momentum
        shape = [1] * P_x.dim
        shape[1] = int(num_features)
        kw = dict(device=device, dtype=dtype)
        self.gamma = torch.nn.Parameter(torch.ones(shape, **kw)) if affine else None
        self.beta = torch.nn.Parameter(torch.zeros(shape, **kw)) if affine else None
        self.track = track_running_stats
        if track_running_stats:
            self.register_buffer("running_mean", torch.zeros(shape, **kw))
            self.register_buffer("running_var", torch.ones(shape, **kw))
            self.register_buffer("num_batches_tracked", torch.zeros((), dtype=torch.long, device=device))

    def forward(self, x):
        axes = [d for d in range(x.dim()) if d != 1]
        if self.training or not self.track:
            s = torch.stack([x.sum(axes, keepdim=True), (x * x).sum(axes, keepdim=True),
                             torch.full_like(x.sum(axes, keepdim=True), x.numel() // x.shape[1])])
            if _on():
                s = s.clone()
                dist.all_reduce(s)            # statistics only; gradients of the statistics stay local
            mean = s[0] / s[2]
            var = (s[1] / s[2] - mean * mean).clamp_min(0)
            if self.track and self.training:
                with torch.no_grad():
                    self.running_mean.lerp_(mean, self.momentum)
                    self.running_var.lerp_(var * s[2] / (s[2] - 1).clamp_min(1), self.momentum)
                    self.num_batches_tracked += 1
        else:
            mean, var = self.running_mean, self.running_var
        y = (x - mean) * torch.rsqrt(var + self.eps)
        return y * self.gamma + self.beta if self.gamma is not None else y
