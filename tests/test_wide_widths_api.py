"""Widths 48 and 64 (WIDE_WIDTHS) on the CPU: which configurations the fused engine accepts, what ``backend="auto"``
chooses, the plan's memory figures and ``tools/plan.py --width``."""
import os
import subprocess
import sys

import pytest
import torch

from dfno_b200.models.fused import (HBM_BUDGET, SUPPORTED_WIDTHS, WIDE_WIDTHS, EnginePlan, supports, wants)
from dfno_b200.parallel.partition import Partition

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GIB = 2 ** 30


def P(*shape):
    n = 1
    for v in shape:
        n *= v
    return Partition(list(range(n)), list(shape))


def test_width_sets():
    assert SUPPORTED_WIDTHS == (4, 8, 12, 16, 20, 24, 32)
    assert WIDE_WIDTHS == (48, 64)


@pytest.mark.parametrize("width", WIDE_WIDTHS)
@pytest.mark.parametrize("grid,in_shape,T,modes", [
    ((1, 1, 1, 2, 1, 1), [1, 1, 128, 128, 128, 1], 20, (12, 12, 12, 10)),     # headline shape on 2 GPUs
    ((1, 1, 1, 1, 1, 1), [1, 1, 60, 60, 64, 1], 30, (12, 12, 12, 8)),         # reference two-phase run
    ((1, 1, 1, 1, 1), [1, 1, 64, 64, 10], 16, (12, 12, 8)),                   # reference Navier-Stokes, 2-D + time
    ((1, 1, 1, 1, 1, 1), [1, 1, 32, 32, 32, 1], 16, (4, 4, 4, 4)),
], ids=["headline_2gpu", "two_phase", "navier_stokes", "small"])
def test_wide_widths_accepted_on_round2_shapes(grid, in_shape, T, modes, width):
    ok, why = supports(P(*grid), in_shape, T, width, modes)
    assert ok, why
    if len(grid) == 1 or grid.count(1) == len(grid):
        assert wants((P(*grid), in_shape, T, width, modes), {"device": "cuda", "dtype": torch.bfloat16}, "auto")


@pytest.mark.parametrize("width", WIDE_WIDTHS)
def test_wide_widths_refused_off_round2(width):
    """2 * KZ > 128 (modes_z = 34): the round-1 route, which has no wide-width kernels"""
    in_shape, T, modes = [2, 1, 8, 8, 128, 1], 8, (2, 2, 34, 3)
    ok, why = supports(P(1, 1, 1, 1, 1, 1), in_shape, T, width, modes)
    assert not ok and f"width {width}" in why and "round-2" in why, why
    assert supports(P(1, 1, 1, 1, 1, 1), in_shape, T, 32, modes)[0]
    assert not wants((P(1, 1, 1, 1, 1, 1), in_shape, T, width, modes),
                     {"device": "cuda", "dtype": torch.bfloat16}, "auto")
    with pytest.raises(ValueError, match="round-2"):
        wants((P(1, 1, 1, 1, 1, 1), in_shape, T, width, modes), {"device": "cuda"}, "fused")


@pytest.mark.parametrize("width", WIDE_WIDTHS)
def test_wide_widths_refuse_several_outputs(width):
    ok, why = supports(P(1, 1, 1, 1, 1, 1), [1, 1, 32, 32, 32, 1], 16, width, (4, 4, 4, 4), out_channels=2)
    assert not ok and "width" in why and "out_channels = 2" in why, why


@pytest.mark.parametrize("width", [40, 56, 128])
def test_other_widths_still_refused(width):
    ok, why = supports(P(1, 1, 1, 1, 1, 1), [1, 1, 32, 32, 32, 1], 16, width, (4, 4, 4, 4))
    assert not ok and f"width {width} not in {SUPPORTED_WIDTHS}" in why, why


def _plan(in_shape, T, width, modes, world):
    B, Cin, X, Y, Z, Tin = in_shape
    pl = EnginePlan(B, Cin, Tin, width, T, X, Y, Z, modes, world=world, rank=0)
    pl.finish(4)
    return pl


@pytest.mark.parametrize("in_shape,T,width,modes,world,gib", [
    ([1, 1, 128, 128, 128, 1], 20, 64, (12, 12, 12, 10), 1, 122.0),
    ([1, 1, 128, 128, 128, 1], 20, 64, (12, 12, 12, 10), 2, 61.0),
    ([1, 1, 128, 128, 128, 1], 20, 64, (8, 8, 8, 8), 1, 68.6),
    ([1, 1, 60, 60, 64, 1], 30, 64, (12, 12, 12, 8), 1, 63.5),
    ([1, 1, 128, 128, 128, 1], 20, 48, (12, 12, 12, 10), 1, 79.0),
], ids=["w64_1gpu", "w64_2gpu", "w64_modes8", "w64_two_phase", "w48_1gpu"])
def test_memory_at_wide_widths(in_shape, T, width, modes, world, gib):
    pl = _plan(in_shape, T, width, modes, world)
    assert pl.fused_pw
    total = pl.memory_bytes(train=True)["total"] / GIB
    assert abs(total - gib) < 0.06 * gib, total
    ok, why = supports(P(1, 1, 1, world, 1, 1), in_shape, T, width, modes)
    B, _, X, Y, Z, _ = in_shape
    assert ok == (total * GIB <= HBM_BUDGET and B * width * X * (Y // world) * Z * T < 2 ** 31), why


def test_navier_stokes_memory_at_width_64():
    """2-D + time, 64 x 64, 10 steps in, 16 out: a few GiB"""
    pl = EnginePlan(1, 1, 10, 64, 16, 1, 64, 64, (0, 12, 12, 8), world=1, rank=0)
    pl.finish(4)
    assert 1.0 < pl.memory_bytes(train=True)["total"] / GIB < 4.0


def test_segments_at_width_64():
    pl = _plan([1, 1, 128, 128, 128, 1], 20, 64, (12, 12, 12, 10), 2)
    C, Q = 64, pl.Q
    assert pl.segments["linear2.W"][1] == (C, 1) and pl.segments["linear3.W"][1] == (128, C)
    assert pl.segments["blocks.0.linear.W"][1] == (C, C)
    assert pl.segments["blocks.3.spectral"][1] == (C, C, Q, 2)
    assert pl.n_small % 64 == 0 and pl.n_small >= 20 + 20 + 2 * C + 4 * C * C + 128 * C + 128 + 129
    assert pl.n_theta == pl.n_small + 4 * C * C * Q * 2


def test_plan_tool_prints_a_wide_plan():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "plan.py"), "--shape", "128", "128", "128", "20",
                        "--width", "64", "--modes", "12", "12", "12", "10", "--gpus", "2"],
                       capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "64" in r.stdout and len(r.stdout.splitlines()) > 3, r.stdout
