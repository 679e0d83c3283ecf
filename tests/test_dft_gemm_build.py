"""ptxas report and SASS of csrc/dft_gemm_sm90.cu (no GPU needed): the kernel is instantiated per padded operator
width, so that each wgmma chain issues back to back (a width decided per instruction makes ptxas serialise every
wgmma, C7511), with one WARPGROUP.DEPBAR per chain.  Compiled with the extension's own flags."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "dfno_b200", "csrc", "dft_gemm_sm90.cu")


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
        obj = os.path.join(tmp, "dg.o")
        r = subprocess.run([nvcc, *build.NVCC_FLAGS, *inc, "-c", SRC, "-o", obj],
                           capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, r.stderr[-4000:]
        sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", obj],
                              capture_output=True, text=True, timeout=600).stdout
    return r.stdout + r.stderr, sass


def _per_kernel(text):
    """{n_pad: [ptxas lines about it]} for every dft_gemm_kernel instantiation"""
    out, cur = {}, None
    for line in text.splitlines():
        m = re.search(r"dft_gemm_kernelILi(\d+)E", line)
        if m and "Compiling entry function" in line:
            cur = int(m.group(1))
            out.setdefault(cur, [])
        elif m and re.search(r"C75\d\d", line):
            out.setdefault(int(m.group(1)), []).append(line)
        elif cur is not None and ("spill" in line or "stack" in line):
            out[cur].append(line)
    return out


def _body(sass, n):
    fn = re.search(r"Function : \S*dft_gemm_kernelILi%dE\S*\n(.*?)(?=\n\s*Function : |\Z)" % n, sass, re.S)
    assert fn, f"n_pad = {n} missing from the SASS"
    return fn.group(1)


def test_dft_gemm_every_width_is_instantiated(report):
    assert set(_per_kernel(report[0])) == set(range(16, 257, 16)), sorted(_per_kernel(report[0]))


def test_dft_gemm_no_serialised_wgmma(report):
    bad = {w: [l for l in ls if "C7511" in l or "C7520" in l] for w, ls in _per_kernel(report[0]).items()}
    assert not any(bad.values()), {w: len(v) for w, v in bad.items() if v}


# the widest accumulators (128 registers: n_pad = 128 with two m64 halves, n_pad = 240 and 256 with one) still spill a
# few words next to the epilogue's address registers
SPILLING = {128, 240, 256}


def test_dft_gemm_no_spills(report):
    for w, ls in _per_kernel(report[0]).items():
        spills = [l for l in ls if "spill" in l]
        assert spills, w
        if w not in SPILLING:
            assert all(re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", l)
                       for l in spills), (w, spills)


@pytest.mark.parametrize("n,halves", [(48, 2), (256, 1)])
def test_dft_gemm_one_wait_per_chain(report, n, halves):
    """the headline widths: n_pad = 48 (G2, G3, iG1b; 128-row tiles) and 256 (iG3, iG2; 64-row tiles) -- one chain of
    four k16 steps per K block and m64 half, closed by one WARPGROUP.DEPBAR instead of one per HGMMA"""
    body = _body(report[1], n)
    assert body.count("HGMMA") >= 4 * halves and body.count("WARPGROUP.DEPBAR") == 1, (body.count("HGMMA"),
                                                                                        body.count("WARPGROUP.DEPBAR"))
