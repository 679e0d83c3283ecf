"""5 <= Cin <= 16 input channels on the fused engine (no GPU needed): eligibility on both routes, the refusals that
stay, the traffic model's lift entries and tools/plan.py."""
import os
import subprocess
import sys

import pytest
import torch

from dfno_b200.models.fused import LIFT_MAX_W, MAX_IN, EnginePlan, supports, wants

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(device=torch.device("cuda"), dtype=torch.bfloat16)


class _Grid:
    def __init__(self, *shape):
        self.shape, self.dim = list(shape), len(shape)


G1 = _Grid(1, 1, 1, 1, 1, 1)
# (route, in_shape with Cin = 1, T, modes): round 2 (2*2*modes_z <= 128) and round 1 (2*2*modes_z = 136)
ROUTES = [("round2", [1, 1, 32, 32, 32, 1], 10, (4, 4, 4, 3)),
          ("round1", [1, 1, 16, 16, 80, 1], 8, (4, 4, 34, 3))]


@pytest.mark.parametrize("width", [4, 20, 32, 64])
@pytest.mark.parametrize("Cin", [5, 8, 16])
@pytest.mark.parametrize("route", ROUTES, ids=[r[0] for r in ROUTES])
def test_many_inputs_are_eligible(route, Cin, width):
    name, shape, T, modes = route
    in_shape = [shape[0], Cin, *shape[2:]]
    ok, why = supports(G1, in_shape, T, width, modes)
    if name == "round1" and width == 64:           # the wide widths have no round-1 kernels, whatever Cin is
        assert not ok and "round-2 route" in why, why
        assert supports(G1, [shape[0], 1, *shape[2:]], T, width, modes)[1] == why
        return
    assert ok, why
    assert wants((G1, in_shape, T, width, modes), KW, "auto")
    assert wants((G1, in_shape, T, width, modes), KW, "fused")


def test_more_than_sixteen_inputs_are_refused():
    assert MAX_IN == 16
    for width in (20, 64):
        ok, why = supports(G1, [1, 17, 32, 32, 32, 1], 10, width, (4, 4, 4, 3))
        assert not ok and "16" in why, why
        assert not wants((G1, [1, 17, 32, 32, 32, 1], 10, width, (4, 4, 4, 3)), KW, "auto")
        with pytest.raises(ValueError, match="Cin <= 16"):
            wants((G1, [1, 17, 32, 32, 32, 1], 10, width, (4, 4, 4, 3)), KW, "fused")
    ok, why = supports(G1, [1, 8, 32, 32, 32, 65], 10, 20, (4, 4, 4, 3))
    assert not ok and "Tin <= 64" in why, why
    # 2-D + time
    assert supports(_Grid(1, 1, 1, 1, 1), [2, 16, 32, 32, 10], 16, 20, (4, 4, 4))[0]
    assert not supports(_Grid(1, 1, 1, 1, 1), [2, 17, 32, 32, 10], 16, 20, (4, 4, 4))[0]


def test_lift_budget_still_refuses_large_cin_times_width():
    """T*Tin + T + 2*(C*Cin + C) <= kLiftMaxW: at width 64 and 16 inputs the W2 terms alone take 2176 floats"""
    C, Cin = 64, 16
    ok_T = (LIFT_MAX_W - 2 * (C * Cin + C)) // (64 + 1)
    g = _Grid(1, 1, 1, 1, 1, 1)
    shape = [1, Cin, 16, 16, 16, 64]
    assert supports(g, shape, ok_T - ok_T % 2, C, (2, 2, 4, 4))[0]
    bad_T = ok_T + 2 - ok_T % 2
    need = bad_T * 64 + bad_T + 2 * (C * Cin + C)
    assert need > LIFT_MAX_W
    ok, why = supports(g, shape, bad_T, C, (2, 2, 4, 4))
    assert not ok and "kLiftMaxW" in why and str(need) in why, why
    # the same T and Tin fit with fewer inputs: the budget, not the channel bound, refused it
    assert supports(g, [1, 1, 16, 16, 16, 64], bad_T, C, (2, 2, 4, 4))[0]


def test_cost_model_lift_entries_count_the_input():
    pl1 = EnginePlan(1, 1, 1, 20, 20, 128, 128, 128, (12, 12, 12, 10))
    pl1.finish(4)
    pl16 = EnginePlan(1, 16, 10, 20, 20, 128, 128, 128, (12, 12, 12, 10))
    pl16.finish(4)
    act = pl1.n_act * 2
    for pl, cin, tin in ((pl1, 1, 1), (pl16, 16, 10)):
        st = {n: b for n, _, b, _ in pl.cost_model()["stages"]}
        x_bytes = 128 ** 3 * cin * tin * 4
        assert st["lift fwd"] == act + x_bytes and st["lift bwd"] == act + x_bytes
    assert abs(128 ** 3 * 4 - 8.4e6) < 0.1e6           # headline input: 8.4 MB per lift call
    x16 = 128 ** 3 * 16 * 10 * 4
    assert 0.75 < x16 / act < 0.85                      # Cin = 16, Tin = 10: the input is close to the size of h
    assert pl16.memory_bytes()["input_output"] - pl1.memory_bytes()["input_output"] == x16 - 128 ** 3 * 4


def test_plan_tool_reports_an_eligible_plan_at_16_inputs():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "plan.py"), "--shape", "128", "128", "128", "20",
                        "--modes", "12", "12", "12", "10", "--in-channels", "16", "--in-timesteps", "10"],
                       capture_output=True, text=True, cwd=ROOT, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "fused engine: yes" in r.stdout, r.stdout
    assert "in_shape = [1, 16, 128, 128, 128, 10]" in r.stdout, r.stdout
