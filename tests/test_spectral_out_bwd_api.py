"""The folded adjoint spectral_out without a GPU: the traffic model's ``fold_bwd`` keyword and the shapes the kernel
takes (spectral_out_adj_check)."""
from dfno_b200.models.fused import EnginePlan


def _plan(nb):
    pl = EnginePlan(1, 1, 1, 20, 20, 128, 128, 128, (12, 12, 12, 10), world=1, rank=0)
    pl.finish(nb)
    return pl


def test_cost_model_fold_bwd_saves_two_activation_passes_per_block_above_the_first():
    act = _plan(4).n_act * 2
    for nb in (1, 2, 3, 4):
        pl = _plan(nb)
        base, fold = pl.cost_model(), pl.cost_model(fold_bwd=True)
        assert base["hbm_bytes"] - fold["hbm_bytes"] == (2 * nb - 2) * act, nb
        calls = {n: c for n, c, _, _ in fold["stages"]}
        if nb == 1:
            assert fold == base
        else:
            assert calls["dpre_dw"] == 1 and "spectral_out adj" not in calls
            assert calls["spectral_out adj+dpre"] == 1 and calls["spectral_out adj+dW"] == 1
            assert calls["spectral_out adj+dpre+dW"] == nb - 2
    # the headline step: 24 -> 18 activation passes in the backward's pointwise tail, about 10 GB
    pl = _plan(4)
    assert abs(pl.cost_model()["hbm_bytes"] - pl.cost_model(fold_bwd=True)["hbm_bytes"] - 10.07e9) < 0.01e9
    # the default keeps the stages it had
    st = {n: (c, b) for n, c, b, _ in pl.cost_model()["stages"]}
    assert st["spectral_out adj"][0] == 4 and st["dpre_dw"] == (4, 4 * act)


def test_check_refuses_only_what_does_not_fit():
    from dfno_b200.ops import build
    ok = build.load().spectral_out_adj_check
    # (n_pad, k_pad, C, Z, K1, dpre, dw)
    for C in (4, 8, 20, 32, 48, 64):
        for Z in (64, 96, 128, 256):
            for K1 in (24, 48, 64):
                assert ok(Z, 64, C, Z, K1, True, True) == "", (C, Z, K1)
            assert ok(Z, 128, C, Z, 128, True, False) == "" and ok(Z, 128, C, Z, 128, False, True) == ""
    assert ok(128, 128, 20, 128, 128, True, True) == ""       # two U blocks: 226 of 227 KB
    # the middle-block variant with two U blocks and Z > 128: the operator plus two stages exceed shared memory
    assert "shared memory" in ok(144, 128, 20, 144, 128, True, True)
    assert "shared memory" in ok(256, 128, 20, 256, 128, True, True)
    assert ok(128, 64, 20, 128, 24, False, False) != ""
    assert ok(128, 64, 20, 100, 24, True, True) != ""         # Z % 8


def test_folded_adjoint_instantiations_do_not_spill():
    """ptxas report of spectral_out_sm90.cu with the extension's own flags: the three folded adjoint kernels keep
    their values in registers."""
    import os
    import re
    import shutil
    import subprocess
    import tempfile

    import pytest
    import torch.utils.cpp_extension as ext

    from dfno_b200.ops import build
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    nvcc = nvcc if os.path.exists(nvcc) else shutil.which("nvcc")
    if nvcc is None:
        pytest.skip("nvcc not found")
    inc = [f"-I{p}" for p in [build.CSRC] + ext.include_paths()]
    with tempfile.TemporaryDirectory() as tmp:
        p = subprocess.run([nvcc, *build.NVCC_FLAGS, *inc, "-c", os.path.join(build.CSRC, "spectral_out_sm90.cu"),
                            "-o", os.path.join(tmp, "so.o")], capture_output=True, text=True, timeout=3000)
    text = p.stdout + p.stderr
    assert p.returncode == 0, text[-4000:]
    per, cur = {}, None
    for line in text.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            per[cur] = []
        elif cur is not None and "spill" in line:
            per[cur].append(line)
    found = {k: v for k, v in per.items() if re.search(r"spectral_out_adj_kernelILb[01]ELb[01]E", k)}
    assert len(found) == 3, sorted(found)
    for k, lines in found.items():
        assert lines, k
        for l in lines:
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", l)
            assert m and int(m.group(1)) == 0 and int(m.group(2)) == 0, (k, l)
