"""FusedAdam as a ``torch.optim.Optimizer`` (argument checks, schedulers, state dicts) and the training scripts'
optimizer flags, without a GPU: the optimizer is built on a model stub that holds only ``theta``."""
import argparse
import math
import os
import subprocess
import sys
import types
import warnings

import pytest
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPTS = ["training/navier_stokes/experiment_navier_stokes.py", "training/two_phase/train_two_phase.py"]


def _stub(n=10):
    return types.SimpleNamespace(theta=nn.Parameter(torch.zeros(n)))


def _opt(**kw):
    from dfno_b200.models.fused import FusedAdam
    return FusedAdam(_stub(), **kw)


@pytest.mark.parametrize("kw", [dict(lr=-1e-3), dict(eps=-1.0), dict(betas=(1.0, 0.999)), dict(betas=(0.9, -0.1)),
                                dict(betas=(0.9,)), dict(weight_decay=-1e-4), dict(max_grad_norm=0.0),
                                dict(max_grad_norm=-1.0), dict(max_grad_norm=math.nan)])
def test_invalid_arguments_raise(kw):
    with pytest.raises(ValueError):
        _opt(**kw)


def test_setting_an_invalid_max_grad_norm_raises():
    opt = _opt(max_grad_norm=1.0)
    with pytest.raises(ValueError):
        opt.max_grad_norm = 0.0
    opt.max_grad_norm = math.inf                  # measure the norm, do not clip
    opt.max_grad_norm = None


def test_is_a_torch_optimizer_with_one_group():
    opt = _opt(lr=2e-3, betas=(0.8, 0.99), eps=1e-7, weight_decay=1e-4)
    assert isinstance(opt, torch.optim.Optimizer)
    assert len(opt.param_groups) == 1 and opt.param_groups[0]["params"][0] is opt.model.theta
    with pytest.raises(ValueError):
        opt.add_param_group({"params": [nn.Parameter(torch.zeros(3))]})
    g = opt.param_groups[0]
    assert (opt.lr, opt.betas, opt.eps, opt.weight_decay) == (2e-3, (0.8, 0.99), 1e-7, 1e-4)
    assert g["decoupled_weight_decay"] is False and g["max_grad_norm"] is None
    opt.lr = 5e-4                                 # attributes and the group are one thing
    assert g["lr"] == 5e-4
    g["betas"] = (0.5, 0.9)
    assert opt.betas == (0.5, 0.9)
    # the defaults keep the host-argument kernel path; a graph captured on it depends on these values
    assert not opt.device_hparams()
    assert opt.graph_key() == ("host", 5e-4, (0.5, 0.9), 1e-7, 1e-4)
    assert _opt(decoupled_weight_decay=True).device_hparams() and _opt(max_grad_norm=1.0).device_hparams()
    assert _opt(max_grad_norm=1.0).graph_key() == ("device", True)
    opt.use_device_hparams()                      # what the Trainer does when a captured host argument changes
    assert opt.device_hparams() and opt.graph_key() == ("device", False)


def _schedulers():
    S = torch.optim.lr_scheduler
    return {
        "step": lambda o: S.StepLR(o, step_size=3, gamma=0.5),
        "cosine": lambda o: S.CosineAnnealingLR(o, T_max=10),
        "warmup": lambda o: S.LambdaLR(o, lambda k: min(1.0, (k + 1) / 4)),
        "onecycle": lambda o: S.OneCycleLR(o, max_lr=1e-2, total_steps=12),
        "onecycle_nomom": lambda o: S.OneCycleLR(o, max_lr=1e-2, total_steps=12, cycle_momentum=False),
    }


@pytest.mark.parametrize("name", list(_schedulers()))
def test_schedulers_drive_the_group_as_for_torch_adam(name):
    make = _schedulers()[name]
    opt = _opt(lr=1e-3)
    ref = torch.optim.Adam([nn.Parameter(torch.zeros(10))], lr=1e-3)
    s, r = make(opt), make(ref)
    assert opt.device_hparams(), "an attached scheduler moves the step to device hyperparameters"
    with warnings.catch_warnings():
        warnings.simplefilter("error")            # no "scheduler.step() before optimizer.step()"
        for _ in range(11):
            opt.step()                            # theta.grad is None: nothing to update
            ref.step()
            s.step()
            r.step()
            assert opt.lr == ref.param_groups[0]["lr"] and opt.betas == ref.param_groups[0]["betas"]


def test_old_state_dict_loads_as_plain_adam():
    opt = _opt(lr=1e-3, decoupled_weight_decay=True, max_grad_norm=2.0)
    old = {"m": torch.full((10,), 0.5), "v": torch.full((10,), 0.25), "step": 7, "lr": 3e-4,
           "betas": [0.9, 0.95], "eps": 1e-6, "weight_decay": 1e-4}           # as written before this change
    opt.load_state_dict(old)
    assert opt.step_count == 7 and float(opt.step_dev) == 7.0
    assert torch.equal(opt.m, old["m"]) and torch.equal(opt.v, old["v"])
    assert (opt.lr, opt.betas, opt.eps, opt.weight_decay) == (3e-4, (0.9, 0.95), 1e-6, 1e-4)
    assert opt.decoupled_weight_decay is False and opt.max_grad_norm is None and not opt.device_hparams()


def test_state_dict_round_trip_with_a_scheduler():
    opt = _opt(lr=1e-3, weight_decay=1e-2, decoupled_weight_decay=True, max_grad_norm=1.5)
    sched = torch.optim.lr_scheduler.StepLR(opt, step_size=2, gamma=0.1)
    for _ in range(5):
        opt.step()
        sched.step()
    sd, ssd = opt.state_dict(), sched.state_dict()
    for k in ("m", "v", "step", "lr", "betas", "eps", "weight_decay", "decoupled_weight_decay", "max_grad_norm"):
        assert k in sd
    opt2 = _opt(lr=1.0)
    opt2.load_state_dict(sd)
    sched2 = torch.optim.lr_scheduler.StepLR(opt2, step_size=2, gamma=0.1, last_epoch=-1)
    sched2.load_state_dict(ssd)
    assert opt2.param_groups[0]["initial_lr"] == 1e-3
    assert (opt2.lr, opt2.decoupled_weight_decay, opt2.max_grad_norm) == (opt.lr, True, 1.5)
    opt.step(); sched.step(); opt2.step(); sched2.step()
    assert opt2.lr == opt.lr


def test_checkpoint_round_trips_a_scheduler(tmp_path):
    import dfno_b200 as d
    _, P_x, _ = d.create_standard_partitions((1, 1, 1, 1, 1, 1))
    net = d.DistributedFNO(P_x, [1, 1, 8, 8, 8, 1], 4, 4, (2, 2, 2, 2), num_blocks=1, device=torch.device("cpu"),
                           dtype=torch.float32, backend="torch")
    params = [p for p in net.parameters() if p.numel()]
    opt = torch.optim.Adam(params, lr=1e-3)
    sched = torch.optim.lr_scheduler.StepLR(opt, step_size=2, gamma=0.5)
    for _ in range(5):
        opt.step()
        sched.step()
    d.save_checkpoint(net, str(tmp_path), epoch=5, optimizer=opt, scheduler=sched)
    opt2 = torch.optim.Adam(params, lr=1e-3)
    sched2 = torch.optim.lr_scheduler.StepLR(opt2, step_size=2, gamma=0.5)
    d.load_checkpoint(net, str(tmp_path), epoch=5, optimizer=opt2, scheduler=sched2, restore_rng=False)
    assert sched2.last_epoch == sched.last_epoch == 5 and opt2.param_groups[0]["lr"] == opt.param_groups[0]["lr"]
    # files written without a scheduler (or before this change) still load
    d.save_checkpoint(net, str(tmp_path), epoch=6, optimizer=opt)
    d.load_checkpoint(net, str(tmp_path), epoch=6, optimizer=opt2, scheduler=sched2, restore_rng=False)


# ------------------------------------------------------------------ script flags
def _args(argv):
    import dfno_b200 as d
    return d.add_optimizer_args(argparse.ArgumentParser()).parse_args(argv)


def test_flag_defaults_keep_todays_optimizer():
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedAdam
    args = _args([])
    assert (args.lr_step_size, args.clip_grad_norm, args.decoupled_weight_decay) == (None, None, False)
    # Navier-Stokes: Adam(1e-3, weight_decay 1e-4); two-phase: Adam(lr)
    opt, sched, clip = d.make_optimizer(_stub(), args, fused=True, lr=1e-3, weight_decay=1e-4)
    assert isinstance(opt, FusedAdam) and sched is None and clip is None
    assert (opt.lr, opt.weight_decay, opt.decoupled_weight_decay, opt.max_grad_norm) == (1e-3, 1e-4, False, None)
    assert not opt.device_hparams()
    net = nn.Linear(3, 2)
    opt, sched, clip = d.make_optimizer(net, args, fused=False, lr=1e-3, weight_decay=1e-4)
    assert type(opt) is torch.optim.Adam and sched is None and clip is None
    g = opt.param_groups[0]
    assert (g["lr"], g["weight_decay"], g["decoupled_weight_decay"]) == (1e-3, 1e-4, False)


def test_flags_select_schedule_decay_and_clipping():
    import dfno_b200 as d
    args = _args(["--lr-step-size", "100", "--lr-gamma", "0.5", "--clip-grad-norm", "1.0",
                  "--decoupled-weight-decay"])
    opt, sched, clip = d.make_optimizer(_stub(), args, fused=True, lr=1e-3, weight_decay=1e-4)
    assert isinstance(sched, torch.optim.lr_scheduler.StepLR) and (sched.step_size, sched.gamma) == (100, 0.5)
    assert opt.max_grad_norm == 1.0 and opt.decoupled_weight_decay and clip is None
    net = nn.Linear(3, 2)
    opt, sched, clip = d.make_optimizer(net, args, fused=False, lr=1e-3)
    assert opt.param_groups[0]["decoupled_weight_decay"] and isinstance(sched, torch.optim.lr_scheduler.StepLR)
    for p in net.parameters():
        p.grad = torch.full_like(p, 10.0)
    norm = clip()
    assert float(norm) == pytest.approx(10.0 * math.sqrt(8))
    total = math.sqrt(sum(float((p.grad ** 2).sum()) for p in net.parameters()))
    assert total == pytest.approx(1.0, rel=1e-5)


@pytest.mark.parametrize("script", SCRIPTS)
def test_scripts_take_the_flags(script):
    r = subprocess.run([sys.executable, os.path.join(ROOT, script), "--help"], capture_output=True, text=True,
                       cwd=ROOT, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    for flag in ("--lr-step-size", "--lr-gamma", "--clip-grad-norm", "--decoupled-weight-decay"):
        assert flag in r.stdout, (flag, r.stdout[-2000:])
