"""``input_grad``: the constructor keyword that asks the fused engine for dL/dx (CPU only).  The portable backend
accepts it and always differentiates its input; ``DistributedFNO``'s backend dispatch hands it to the engine."""
import pytest
import torch

import dfno_b200 as d
from dfno_b200.models import fused


def test_portable_backend_accepts_input_grad_and_differentiates_x():
    _, P_x, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    torch.manual_seed(0)
    shape = [1, 1, 8, 8, 8, 1]
    net = d.DistributedFNO(P_x, shape, 4, 4, (2, 2, 2, 2), num_blocks=1, input_grad=True, backend="torch")
    assert not isinstance(net, fused.FusedDistributedFNO)
    x = torch.randn(*shape, requires_grad=True)
    (dx,) = torch.autograd.grad(net(x).square().sum(), x)
    assert dx.shape == x.shape and dx.dtype == x.dtype and float(dx.abs().max()) > 0


def test_backend_dispatch_passes_input_grad_to_the_fused_engine(monkeypatch):
    _, P_x, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    args = (P_x, [1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3))
    kw = dict(device=torch.device("cuda"), dtype=torch.bfloat16)
    # the keyword does not change which backend serves a configuration
    assert fused.wants(args, dict(kw, input_grad=True), "auto") == fused.wants(args, kw, "auto") is True
    assert fused.wants(args, dict(kw, input_grad=True, device=torch.device("cpu")), "auto") is False
    seen = {}

    class Engine(fused.FusedDistributedFNO):
        def __init__(self, *a, **k):          # records what the dispatch hands over (no GPU needed)
            torch.nn.Module.__init__(self)
            seen.update(k)

    monkeypatch.setattr(fused, "FusedDistributedFNO", Engine)
    net = d.DistributedFNO(*args, input_grad=True, **kw)
    assert isinstance(net, Engine) and seen.get("input_grad") is True


def test_input_grad_is_a_keyword_of_both_constructors():
    import inspect
    for cls in (d.DistributedFNO, fused.FusedDistributedFNO):
        p = inspect.signature(cls.__init__).parameters["input_grad"]
        assert p.default is False, cls


def test_fused_engine_refuses_input_gradients_without_the_keyword():
    """The refusal (and its message) of an engine built without input_grad, checked without a GPU."""
    class Eng:
        input_grad = False
    x = torch.zeros(2, requires_grad=True)
    with pytest.raises(RuntimeError, match="input gradients.*input_grad=True"):
        fused._FusedFn.apply(x, torch.zeros(1), Eng(), False)
