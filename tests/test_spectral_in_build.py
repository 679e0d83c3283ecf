"""ptxas report and SASS of csrc/spectral_in_sm90.cu (no GPU needed): the wgmma chains of spectral_in must issue back
to back.  A width decided per instruction makes ptxas serialise them (C7511: every wgmma waits for the one before it,
22 full wgmma latencies per tile at the headline shape).  Compiled with the extension's own flags."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "dfno_b200", "csrc", "spectral_in_sm90.cu")


def _nvcc():
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = os.path.join(cuda, "bin", "nvcc")
    return exe if os.path.exists(exe) else shutil.which("nvcc")


@pytest.fixture(scope="module")
def report():
    """(ptxas report, SASS of the object)"""
    from dfno_b200.ops import build
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    import torch.utils.cpp_extension as ext
    inc = [f"-I{p}" for p in [build.CSRC] + ext.include_paths()]
    with tempfile.TemporaryDirectory() as tmp:
        obj = os.path.join(tmp, "si.o")
        r = subprocess.run([nvcc, *build.NVCC_FLAGS, *inc, "-c", SRC, "-o", obj],
                           capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, r.stderr[-4000:]
        sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", obj],
                              capture_output=True, text=True, timeout=600).stdout
    return r.stdout + r.stderr, sass


def _per_kernel(text):
    """{(N1, N2): [ptxas lines about it]} for every spectral_in_kernel instantiation"""
    out, cur = {}, None
    for line in text.splitlines():
        m = re.search(r"spectral_in_kernelILi(\d+)ELi(\d+)E", line)
        if m and "Compiling entry function" in line:
            cur = (int(m.group(1)), int(m.group(2)))
            out.setdefault(cur, [])
        elif m and ("C7519" in line or "C7511" in line):
            out.setdefault((int(m.group(1)), int(m.group(2))), []).append(line)
        elif cur is not None and "spill" in line:
            out[cur].append(line)
    return out


def test_spectral_in_every_width_is_instantiated(report):
    k = _per_kernel(report[0])
    assert set(k) == {(n1, n2) for n1 in range(16, 129, 16) for n2 in (16, 32, 48, 64, 80, 128)}, sorted(k)


def test_spectral_in_no_serialised_wgmma(report):
    bad = {w: [l for l in ls if "C7511" in l] for w, ls in _per_kernel(report[0]).items()}
    assert not any(bad.values()), {w: len(v) for w, v in bad.items() if v}


# the widest accumulators (128 registers: N1 = 128 with N2 >= 80, or N2 = 128, i.e. 64 z modes or more than 40 t
# modes) still spill with one consumer warpgroup
SPILLING = {(128, 128), (128, 80), (112, 128), (96, 128), (80, 128)}


def test_spectral_in_no_spills(report):
    for w, ls in _per_kernel(report[0]).items():
        spills = [l for l in ls if "spill" in l]
        assert spills, w
        if w not in SPILLING:
            assert all(re.search(r"\b0 bytes spill stores, 0 bytes spill loads", l) for l in spills), (w, spills)


def test_spectral_in_headline_one_wait_per_chain(report):
    """(n1_pad, n2_pad) = (48, 32), the flagship shape (24 z modes, 10 t modes): four chains (MMA1 / MMA2, one or two
    m64 halves), one WARPGROUP.DEPBAR each, instead of one per HGMMA"""
    sass = report[1]
    fn = re.search(r"Function : \S*spectral_in_kernelILi48ELi32E\S*\n(.*?)(?=\n\s*Function : |\Z)", sass, re.S)
    assert fn, "headline instantiation missing from the SASS"
    body = fn.group(1)
    assert body.count("HGMMA") >= 24 and body.count("WARPGROUP.DEPBAR") == 4, (body.count("HGMMA"),
                                                                              body.count("WARPGROUP.DEPBAR"))
