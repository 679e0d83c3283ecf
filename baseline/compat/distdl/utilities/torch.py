"""``distdl.utilities.torch`` (star-imported by the reference, which relies on ``np`` / ``torch``
leaking through it: reference ``dfno/utils.py:8-9,80``)."""
import numpy as np                                          # noqa: F401
import torch                                                # noqa: F401


class TensorStructure:
    """Shape / dtype / requires_grad record of a tensor (the reference only sets ``.shape``)."""

    def __init__(self, tensor=None):
        self.shape = None
        self.dtype = None
        self.requires_grad = None
        if tensor is not None:
            self.shape = tuple(tensor.shape)
            self.dtype = tensor.dtype
            self.requires_grad = tensor.requires_grad


def zero_volume_tensor(b=None, dtype=None, requires_grad=False, device=None):
    """The "this worker owns nothing" placeholder: an empty tensor (``[b, 0]`` when a batch size is given)."""
    shape = (0,) if b is None else (int(b), 0)
    return torch.empty(*shape, dtype=dtype, requires_grad=requires_grad, device=device)
