"""spectral_in alone (csrc/spectral_in_sm90.cu: truncated z-DFT, t-DFT and the pencil-transpose store in one kernel) at
the headline shape (BC 20, X 128, Y 128, T 20, Z 128, modes mz 12, mt 10) and at the local shapes of a 2, 4 and 8-rank
run (Yl = 64 / 32 / 16), timed with CUDA events against the bytes it must move (the spectral_in entry of the engine's
traffic model, EnginePlan.cost_model(front=True), per call).  The P destination ranks of a multi-rank run are P
buffers on this one GPU, laid out as the engine lays them out (direct S1 below 8 ranks, the staged S1s at 8).
Prints one line per shape and one JSON line; writes nothing.

    python benchmarks/spectral_in_bench.py [--iters 50] [--warmup 5]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from benchmarks.head_bench import gpu_state, time_ms  # noqa: E402
from dfno_b200.models.fused import H100_COPY_GBS, EnginePlan  # noqa: E402
from dfno_b200.ops import build  # noqa: E402
from dfno_b200.ops import operators as OPS  # noqa: E402
from dfno_b200.ops.gemm import pad_operator  # noqa: E402

BC, X, Y, T, Z, MZ, MT = 20, 128, 128, 20, 128, 12, 10


def case(C_, P, iters, warmup, dev):
    pl = EnginePlan(1, 1, 1, BC, T, X, Y, Z, (12, 12, MZ, MT), world=P, rank=0)
    pl.finish(4)
    _, _, need, _ = next(s for s in pl.cost_model(front=True)["stages"] if s[0] == "spectral_in")   # bytes per call
    Yl, KZ, kzl = pl.Yl, pl.KZ, pl.kzl
    p1 = pad_operator(OPS.fwd_real_to_complex(Z, MZ), device=dev)
    p2 = pad_operator(OPS.fwd_complex(T, MT, False), device=dev)
    g = torch.Generator(device=dev).manual_seed(0)
    h = torch.randn(BC, X, Yl, T, Z, device=dev, generator=g).to(torch.bfloat16)
    if pl.staged:                                                # S1s[bc, kz', kt, r_src, x, y_loc, ri]
        dstr, off = [Yl * 2, P * X * Yl * 2, MT * P * X * Yl * 2, kzl * MT * P * X * Yl * 2], 0
    else:                                                        # S1[bc, kz', kt, x, y, ri]
        dstr, off = [Y * 2, X * Y * 2, MT * X * Y * 2, kzl * MT * X * Y * 2], 0
    bufs = [torch.empty(pl.n_S1, device=dev, dtype=torch.bfloat16) for _ in range(P)]
    ptrs = [b.data_ptr() for b in bufs]
    cfg = C_.spectral_in_config(p1.shape[0], p1.shape[1], p2.shape[0], p2.shape[1], P, off, dstr, BC, X, Yl, T, Z, KZ, MT)

    def run():
        C_.spectral_in(h, p1, p2, ptrs, off, dstr, BC, X, Yl, T, Z, KZ, MT)

    ms = time_ms(run, iters, warmup)
    gbs = need / ms / 1e6
    return {"P": P, "Yl": Yl, "staged": pl.staged, "cfg": list(cfg), "ms": round(ms, 4), "bytes": need,
            "gbs": round(gbs, 1), "frac_copy": round(gbs / H100_COPY_GBS, 3)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spectral_in_bench.py needs a GPU")
    C_ = build.load()
    dev = torch.device("cuda", 0)
    rows = []
    for P in (1, 2, 4, 8):
        r = case(C_, P, a.iters, a.warmup, dev)
        rows.append(r)
        print(f"P {P}  Yl {r['Yl']:3d}  cfg {r['cfg']}  {r['ms']:8.3f} ms  {r['bytes'] / 1e9:6.3f} GB  "
              f"{r['gbs']:7.1f} GB/s  {r['frac_copy']:5.1%} of copy")
    state = gpu_state()
    print(f"{state['gpu']}, power limit {state['power_limit_w']} W, SM clock {state['sm_clock_mhz']} MHz "
          f"(max {state['sm_clock_max_mhz']})")
    print(json.dumps({"shape": {"BC": BC, "X": X, "Y": Y, "T": T, "Z": Z, "mz": MZ, "mt": MT}, "iters": a.iters,
                      **state, "copy_gbs": H100_COPY_GBS, "cases": rows}))


if __name__ == "__main__":
    main()
