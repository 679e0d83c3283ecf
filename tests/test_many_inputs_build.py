"""ptxas report of the many-input (5 <= Cin <= 16) lift kernels (no GPU needed): every instantiation is compiled, there
is one per (x dtype, channel bound 8 / 16, Tin == 1, dx) and not one per Cin value, and none spills.  Compiled with
the extension's own flags."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "dfno_b200", "csrc", "pointwise.cu")

# (kernel name pattern, how many instantiations there are)
MANY = [
    (r"lift_fwd_many_kernelI(f|13__nv_bfloat16)Li(8|16)ELb[01]E", 8),
    (r"lift_bwd_many_kernelI(f|13__nv_bfloat16)Li(8|16)ELb[01]ELb[01]E", 16),
]
SPILL_OK = {}                     # no exceptions


def _nvcc():
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = os.path.join(cuda, "bin", "nvcc")
    return exe if os.path.exists(exe) else shutil.which("nvcc")


@pytest.fixture(scope="module")
def report():
    """{kernel: ptxas lines}"""
    from dfno_b200.ops import build
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    import torch.utils.cpp_extension as ext
    inc = [f"-I{p}" for p in [build.CSRC] + ext.include_paths()]
    with tempfile.TemporaryDirectory() as tmp:
        p = subprocess.run([nvcc, *build.NVCC_FLAGS, *inc, "-c", SRC, "-o", os.path.join(tmp, "pointwise.o")],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=3000)
    assert p.returncode == 0, p.stdout[-4000:]
    per, cur = {}, None
    for line in p.stdout.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            per[cur] = []
        elif cur is not None and ("spill" in line or "stack" in line):
            per[cur].append(line)
    return per


@pytest.mark.parametrize("pattern,count", MANY, ids=["lift_fwd_many", "lift_bwd_many"])
def test_many_input_instantiations_do_not_spill(report, pattern, count):
    found = {k: v for k, v in report.items() if re.search(pattern, k)}
    assert len(found) == count, sorted(found)
    for k, lines in found.items():
        spills = [l for l in lines if "spill" in l]
        assert spills, k
        allowed = next((b for p, b in SPILL_OK.items() if re.search(p, k)), 0)
        for l in spills:
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", l)
            assert m and int(m.group(1)) <= allowed and int(m.group(2)) <= allowed, (k, l)


def test_many_input_kernels_are_the_only_new_lift_instantiations(report):
    """the Cin <= 4 kernels keep their 16 forward and 288 backward instantiations; Cin > 4 adds no per-Cin copies"""
    fwd = [k for k in report if re.search(r"lift_fwd_kernelI", k)]
    bwd = [k for k in report if re.search(r"lift_bwd_kernelI", k)]
    assert len(fwd) == 16 and len(bwd) == 288, (len(fwd), len(bwd))
    many = [k for k in report if "many_kernel" in k]
    assert len(many) == sum(c for _, c in MANY)
