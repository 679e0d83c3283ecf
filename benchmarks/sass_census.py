#!/usr/bin/env python
"""SASS instruction census of the built extension (no GPU needed): for every kernel, the number of
instructions and of the mnemonics that prove which hardware paths it uses -- HGMMA (wgmma.mma_async),
WARPGROUP (wgmma fence / commit / wait), UTMALDG / UTMASTG (TMA tensor load / store), SYNCS (mbarrier),
MUFU (special function unit), ATOM/RED, and LDL / STL (local memory: register spills and indexed arrays).

    python benchmarks/sass_census.py --tensor-core > bench_out/sass_census.txt   # only kernels with wgmma / TMA
    python benchmarks/sass_census.py --excerpt dft_gemm_kernel > bench_out/sass_dft_gemm_excerpt.txt
"""
import collections
import os
import re
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

COLS = ["HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UBLKCP", "SYNCS", "HMMA", "MUFU", "STG/ST", "ATOM/RED", "LDL",
        "STL"]
COUNTED = ("HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UBLKCP", "SYNCS", "HMMA", "MUFU", "LDL", "STL")


def excerpt(so: str, kernel: str) -> None:
    """Only the wgmma / TMA / mbarrier / global-store instructions of one kernel."""
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    pat = re.compile(r"UTMA|GMMA|WARPGROUP|SYNCS|\bSTG|\bST\.E|FENCE|MEMBAR|ERRBAR")
    print(f"{kernel} -- wgmma / TMA / mbarrier / global-store instructions "
          f"(full listing: cuobjdump -sass {os.path.relpath(so)}; python benchmarks/sass_census.py --excerpt {kernel})")
    keep = False
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            keep = kernel in m.group(1)
            continue
        if keep and pat.search(line):
            print(line.rstrip())


def main():
    default_so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dfno_b200", "_build",
                              "dfno_b200_C.so")
    if len(sys.argv) > 2 and sys.argv[1] == "--excerpt":
        return excerpt(sys.argv[3] if len(sys.argv) > 3 else default_so, sys.argv[2])
    tc_only = "--tensor-core" in sys.argv
    argv = [a for a in sys.argv if a != "--tensor-core"]
    so = argv[1] if len(argv) > 1 else os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                             "dfno_b200", "_build", "dfno_b200_C.so")
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    counts, order, cur = {}, [], None
    ins = re.compile(r"^\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)")
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur] = collections.Counter()
            order.append(cur)
            continue
        m = ins.match(line)
        if m and cur:
            op = m.group(1)
            c = counts[cur]
            c["inst"] += 1
            base = op.split(".")[0]
            if base in COUNTED:
                c[base] += 1
            elif base in ("STG", "ST"):
                c["STG/ST"] += 1
            elif base in ("ATOM", "ATOMG", "RED", "ATOMS"):
                c["ATOM/RED"] += 1
    names = subprocess.run(["cu++filt"], input="\n".join(order), capture_output=True, text=True).stdout.splitlines()
    print(f"SASS instruction census of the dfno_b200 extension (cuobjdump -sass, sm_90a)")
    print("HGMMA = wgmma.mma_async, WARPGROUP = wgmma fence / commit / wait, UTMALDG/UTMASTG = TMA load/store, "
          "SYNCS = mbarrier ops, LDL/STL = local memory\n")
    print(f"{'kernel':40s} {'inst':>7s} " + " ".join(f"{c:>7s}" for c in COLS))
    for mangled, name in sorted(zip(order, names), key=lambda t: t[1]):
        c = counts[mangled]
        if tc_only and not (c["HGMMA"] or c["UTMALDG"]):
            continue
        short = re.sub(r"\(anonymous namespace\)::|dfno::|<unnamed>::|^void |\((?:int|bool|unsigned int)\)", "", name)
        short = short.split("(")[0]
        print(f"{short[:40]:40s} {c['inst']:7d} " + " ".join(f"{c[k]:7d}" for k in COLS))


if __name__ == "__main__":
    main()
