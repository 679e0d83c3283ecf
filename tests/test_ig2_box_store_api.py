"""The box-store epilogue of the inverse y-DFT (iG2) without a GPU: which plans take it, its tile -> row mapping, the
traffic model's iG2 figure, and the ptxas report of its dft_gemm instantiations."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from dfno_b200.models.fused import EnginePlan
from dfno_b200.ops.gemm import BoxSpec


def _plan(P=1, r=0, B=1, C=20, X=128, Y=128, Z=128, T=20, modes=(12, 12, 12, 10), pad=None):
    pl = EnginePlan(B, 1, 1, C, T, X, Y, Z, modes, world=P, rank=r, pad=pad)
    pl.finish(4)
    return pl


def _ig2(pl, staged=None):
    (st,) = [s for s in pl.chain(staged=pl.staged if staged is None else staged) if s["name"] == "iG2"]
    return st


def test_route_is_chosen_by_the_shape():
    for P in (1, 2, 3, 4, 5, 7):
        assert "box" in _ig2(_plan(P, Y=120 if P in (3, 5, 7) else 128)), P
    assert "box" not in _ig2(_plan(8))                                   # the staged T1s route from 8 ranks on
    assert "box" not in _ig2(_plan(2), staged=True)
    assert "box" not in _ig2(_plan(T=1, modes=(12, 12, 12, 1)))          # T = 1: T1 has no kt pitch
    assert "box" not in _ig2(_plan(modes=(12, 12, 12, 1)))               # mt = 1: 128 KB of staging per warpgroup
    assert "box" in _ig2(_plan(Y=256)) and "box" in _ig2(_plan(X=1, modes=(1, 12, 12, 10)))
    assert "box" in _ig2(_plan(pad=(0, 0, 8, 2)))


def test_launch_descriptors_follow_the_column_parts():
    pl = _plan(Y=256)
    st = _ig2(pl)
    epis = [pl.epi(st, j0, n, spec) for j0, n, spec, _, _ in pl.parts(st)]
    # [mt, mtp, kzl, KZ, Yl, y0, bcx, base_off]: one launch per 128 y, each inside the one destination
    assert [e[0] for e in epis] == [3, 3] and [e[20:] for e in epis] == [[10, 12, 24, 24, 256, 0, 2560, 0],
                                                                         [10, 12, 24, 24, 256, 128, 2560, 0]]
    p2 = _plan(4, 3)
    st = _ig2(p2)
    ((j0, n, spec, p0, pn),) = p2.parts(st)
    assert p2.epi(st, j0, n, spec)[20:] == [10, 12, 6, 24, 32, 0, 2560, 3 * 6 * 12 * 2]
    assert (p0, pn) == (0, None) and st["box"].column_part(0, 128)[1:] == (0, 4)


@pytest.mark.parametrize("mt,kzl,bcx,n", [(10, 24, 3, 128), (10, 8, 2, 64), (7, 24, 5, 128), (10, 4, 3, 128),
                                          (3, 13, 2, 100), (20, 5, 4, 32)])
def test_tiles_cover_every_row_once(mt, kzl, bcx, n):
    box = BoxSpec(mt, (mt + 3) // 4 * 4, kzl, kzl, n, bcx, 0)
    G, rows = box.groups(n), BoxSpec.tile_rows(n)
    assert G == rows // mt
    seen = [0] * (bcx * kzl * mt)
    for row0, live in box.tiles(n):
        assert live % mt == 0 and 0 < live <= G * mt <= rows and row0 % mt == 0
        b = row0 // (kzl * mt)
        assert (row0 + live - 1) // (kzl * mt) == b                      # one bcx per tile
        for i in range(row0, row0 + live):
            seen[i] += 1
    assert seen == [1] * len(seen)
    assert len(box.tiles(n)) == bcx * -(-kzl // G)


def test_headline_tile_count():
    st = _ig2(_plan())
    assert st["box"].groups(128) == 6 and len(st["box"].tiles(128)) == 10240           # 60 of 64 rows used


def test_cost_model_counts_the_padded_t1_write():
    pl = _plan()
    cm = {n: (c, b, l) for n, c, b, l in pl.cost_model(front=True)["stages"]}
    assert cm["iG2"] == (8, (pl.n_T2 + pl.n_T1) * 2, 0)
    assert abs(cm["iG2"][1] - 0.437e9) < 0.001e9
    for P in (2, 4):
        p = _plan(P)
        c = {n: (b, l) for n, _, b, l in p.cost_model()["stages"]}
        assert c["iG2"] == ((p.n_T2 + p.n_T1) * 2, p.n_T1 * 2 * (P - 1) / P)
    p8 = _plan(8)                                                      # staged: the scatter writes the valid part
    c8 = {n: b for n, _, b, _ in p8.cost_model()["stages"]}
    assert c8["iG2"] == (p8.n_T2 + p8.n_T1 // p8.mtp * p8.mt) * 2


# ptxas figures (registers, stack frame, spill stores, spill loads) of every dft_gemm instantiation without the box
# store, as they were before it existed; the box instantiations are separate kernels and must not touch them
BEFORE = {16: (79, 0, 0, 0), 32: (96, 0, 0, 0), 48: (120, 0, 0, 0), 64: (121, 0, 0, 0), 80: (158, 0, 0, 0),
          96: (157, 0, 0, 0), 112: (167, 0, 0, 0), 128: (168, 16, 16, 16), 144: (134, 0, 0, 0), 160: (142, 0, 0, 0),
          176: (150, 0, 0, 0), 192: (156, 0, 0, 0), 208: (168, 0, 0, 0), 224: (168, 0, 0, 0), 240: (168, 8, 16, 16),
          256: (168, 24, 28, 32)}


def test_ptxas_box_instantiations_do_not_spill_and_the_others_are_unchanged():
    import torch.utils.cpp_extension as ext

    from dfno_b200.ops import build
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    nvcc = nvcc if os.path.exists(nvcc) else shutil.which("nvcc")
    if nvcc is None:
        pytest.skip("nvcc not found")
    inc = [f"-I{p}" for p in [build.CSRC] + ext.include_paths()]
    with tempfile.TemporaryDirectory() as tmp:
        p = subprocess.run([nvcc, *build.NVCC_FLAGS, *inc, "-c", os.path.join(build.CSRC, "dft_gemm_sm90.cu"),
                            "-o", os.path.join(tmp, "dg.o")], capture_output=True, text=True, timeout=3000)
    text = p.stdout + p.stderr
    assert p.returncode == 0, text[-4000:]
    got = {}
    for m in re.finditer(r"Function properties for \S*dft_gemm_kernelILi(\d+)ELb([01])E\S*\n\s+(\d+) bytes stack frame, "
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads\n.*?Used (\d+) registers", text):
        got[(int(m.group(1)), m.group(2) == "1")] = tuple(int(m.group(i)) for i in (6, 3, 4, 5))
    assert sorted(got) == sorted((n, b) for n in range(16, 257, 16) for b in (False, True))
    for n in range(16, 257, 16):
        assert got[(n, False)] == BEFORE[n], n
        assert got[(n, True)][1:] == (0, 0, 0), (n, got[(n, True)])
