"""ptxas report of the wide-width (48, 64) instantiations (no GPU needed): every kernel the widths add is compiled and
keeps its values in registers.  Compiled with the extension's own flags."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dfno_b200", "csrc")

# (source, kernel name pattern of the wide instantiations, how many there are)
WIDE = [
    ("spectral.cu", r"mix_fwd_wide_kernelILi(48|64)E", 2),
    ("spectral.cu", r"mix_bwd_wide_kernelILi(48|64)ELb[01]E", 4),
    ("head_sm90.cu", r"head_fwd_kernelILi(64|80)E", 2),
    ("head_sm90.cu", r"head_bwd2_kernelILi(64|80)E", 2),
    ("pointwise.cu", r"lift_bwd_kernelI(f|13__nv_bfloat16)Li(48|64)ELi[1-4]ELb[01]ELb[01]E", 64),
]
# one lift instantiation (bf16 x, Cin = 4, Tin = 1 in registers, with dx, width 64) keeps two words on the stack
SPILL_OK = {r"lift_bwd_kernelI13__nv_bfloat16Li64ELi4ELb1ELb1E": 16}


def _nvcc():
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = os.path.join(cuda, "bin", "nvcc")
    return exe if os.path.exists(exe) else shutil.which("nvcc")


@pytest.fixture(scope="module")
def reports():
    """{source: {kernel: ptxas lines}}"""
    from dfno_b200.ops import build
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    import torch.utils.cpp_extension as ext
    inc = [f"-I{p}" for p in [build.CSRC] + ext.include_paths()]
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        procs = {}
        for src in sorted({w[0] for w in WIDE}):
            procs[src] = subprocess.Popen([nvcc, *build.NVCC_FLAGS, *inc, "-c", os.path.join(CSRC, src), "-o",
                                           os.path.join(tmp, src + ".o")],
                                          stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        for src, p in procs.items():
            text, _ = p.communicate(timeout=3000)
            assert p.returncode == 0, text[-4000:]
            per, cur = {}, None
            for line in text.splitlines():
                m = re.search(r"Compiling entry function '(\S+)'", line)
                if m:
                    cur = m.group(1)
                    per[cur] = []
                elif cur is not None and ("spill" in line or "stack" in line):
                    per[cur].append(line)
            out[src] = per
    return out


@pytest.mark.parametrize("src,pattern,count", WIDE, ids=[w[1].split("I")[0] for w in WIDE])
def test_wide_instantiations_do_not_spill(reports, src, pattern, count):
    found = {k: v for k, v in reports[src].items() if re.search(pattern, k)}
    assert len(found) == count, sorted(found)
    for k, lines in found.items():
        spills = [l for l in lines if "spill" in l]
        assert spills, k
        allowed = next((b for p, b in SPILL_OK.items() if re.search(p, k)), 0)
        for l in spills:
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", l)
            assert m and int(m.group(1)) <= allowed and int(m.group(2)) <= allowed, (k, l)
