import torch


class ZeroVolumeCorrectorFunction(torch.autograd.Function):
    """Loss epilogue: a worker whose loss is zero-volume gets a scalar 0 so that every worker can call
    ``.backward()``; the backward hands an empty gradient back (reference ``dfno/loss.py:35``)."""

    @staticmethod
    def forward(ctx, value):
        ctx.empty_shape = tuple(value.shape) if value.numel() == 0 else None
        if ctx.empty_shape is not None:
            return torch.zeros((), dtype=value.dtype, device=value.device)
        return value.clone()

    @staticmethod
    def backward(ctx, grad):
        if ctx.empty_shape is not None:
            return torch.empty(ctx.empty_shape, dtype=grad.dtype, device=grad.device)
        return grad
