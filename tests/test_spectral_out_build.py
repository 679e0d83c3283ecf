"""ptxas report and SASS of csrc/spectral_out_sm90.cu (no GPU needed): every kernel's wgmma chains have a
compile-time width (chosen once per tile, not per instruction), so ptxas serialises none of them (C7511 / C7520) and
the SASS waits once per chain, not once per HGMMA; and no kernel spills.  Compiled with the extension's own flags."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "dfno_b200", "csrc", "spectral_out_sm90.cu")
KERNELS = [f"spectral_out_kernelILb{g}ELb{p}E" for g, p in ((0, 0), (1, 0), (1, 1))] + \
          [f"spectral_out_adj_kernelILb{d}ELb{w}E" for d, w in ((0, 1), (1, 0), (1, 1))]


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
        obj = os.path.join(tmp, "so.o")
        r = subprocess.run([nvcc, *build.NVCC_FLAGS, *inc, "-c", SRC, "-o", obj],
                           capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, r.stderr[-4000:]
        sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", obj],
                              capture_output=True, text=True, timeout=600).stdout
    return r.stdout + r.stderr, sass


def _per_kernel(text):
    """{kernel: [ptxas lines about it]} for every kernel of the file"""
    out, cur = {}, None
    for line in text.splitlines():
        k = next((k for k in KERNELS if k in line), None)
        if k and "Compiling entry function" in line:
            cur = k
            out.setdefault(cur, [])
        elif k and re.search(r"C75\d\d", line):
            out.setdefault(k, []).append(line)
        elif cur is not None and ("spill" in line or "stack" in line):
            out[cur].append(line)
    return out


def test_every_kernel_is_reported(report):
    assert set(_per_kernel(report[0])) == set(KERNELS), sorted(_per_kernel(report[0]))


def test_no_serialised_wgmma(report):
    bad = {k: [l for l in ls if "C7511" in l or "C7520" in l] for k, ls in _per_kernel(report[0]).items()}
    assert not any(bad.values()), {k: v[:2] for k, v in bad.items() if v}


def test_no_spills(report):
    for k, ls in _per_kernel(report[0]).items():
        spills = [l for l in ls if "spill" in l]
        assert spills and all(re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", l)
                              for l in spills), (k, spills)


@pytest.mark.parametrize("kernel", KERNELS)
def test_one_wait_per_chain(report, kernel):
    """at least four HGMMA per WARPGROUP.DEPBAR (the parent's kernels had one wait per HGMMA)"""
    fn = re.search(r"Function : \S*%s\S*\n(.*?)(?=\n\s*Function : |\Z)" % kernel, report[1], re.S)
    assert fn, f"{kernel} missing from the SASS"
    hgmma, depbar = fn.group(1).count("HGMMA"), fn.group(1).count("WARPGROUP.DEPBAR")
    assert depbar >= 1 and hgmma >= 4 * depbar, (hgmma, depbar)
