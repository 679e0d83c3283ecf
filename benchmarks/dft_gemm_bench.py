"""dft_gemm alone (csrc/dft_gemm_sm90.cu: the resident-operator GEMM of the y / x DFT stages and the inverse t-DFT) per
stage of one spectral convolution -- G2, G3, iG3, iG2 and iG1b, each with the forward and the adjoint chain's operator
-- at the headline shape (BC 20, X 128, Y 128, T 20, Z 128, modes 12 12 12 10) and at the local shapes of a 2, 4 and
8-rank run (Yl = 64 / 32 / 16).  Every stage runs with the engine's own descriptor (EnginePlan.chain(): M, K, lda,
ScatterSpec / ldc, column parts) into destination buffers sized as the engine sizes them; the P destination ranks of a
multi-rank run are P buffers on this one GPU (direct T1 below 8 ranks, the staged T1s at 8).  Timed with CUDA events
against the bytes the stage must move (its entry of EnginePlan.cost_model(front=True), per call).  A stage that runs the
box-store epilogue (iG2 into the direct T1) is also timed with the pair scatter it replaces ("iG2 scatter", against
the valid part of T1 that the scatter writes).
Prints one line per stage and one JSON line; writes nothing.

    python benchmarks/dft_gemm_bench.py [--iters 50] [--warmup 5] [--ranks 1 2 4 8]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from benchmarks.head_bench import gpu_state, time_ms  # noqa: E402
from dfno_b200.models.fused import H100_COPY_GBS, EnginePlan  # noqa: E402
from dfno_b200.ops import build  # noqa: E402
from dfno_b200.ops.gemm import pad_operator  # noqa: E402

BC, X, Y, T, Z, MODES = 20, 128, 128, 20, 128, (12, 12, 12, 10)
STAGES = ("G2", "G3", "iG3", "iG2", "iG1b")


def buffers(pl, dev):
    """the engine's workspaces by stage-descriptor name (bf16 elements, see FusedDistributedFNO.__init__)"""
    n = {"S1": pl.n_S1, "S2": pl.n_S2, "S3": pl.n_S3, "S4": pl.n_S3, "T2": pl.n_T2, "T1": pl.n_T1, "T1s": pl.n_T1,
         "U": pl.n_U}
    g = torch.Generator(device=dev).manual_seed(0)
    return {k: torch.randn(v, device=dev, generator=g).to(torch.bfloat16) for k, v in n.items()}


def cases(C_, P, iters, warmup, dev):
    pl = EnginePlan(1, 1, 1, BC, T, X, Y, Z, MODES, world=P, rank=0)
    pl.finish(4)
    need = {s[0]: s[2] for s in pl.cost_model(front=True)["stages"]}            # bytes per call
    need["iG2 scatter"] = pl.n_T2 * 2 + pl.n_T1 // pl.mtp * pl.mt * 2
    ops = {k: v for k, v in pl.operators().items()}
    bufs = buffers(pl, dev)
    peers = {k: [bufs[k]] + [torch.empty_like(bufs[k]) for _ in range(P - 1)] for k in ("T1", "T1s")}
    rows = []
    variants = []
    for st in pl.chain(staged=pl.staged):
        if st["name"] in STAGES:
            variants.append((st["name"], st))
            if "box" in st:
                variants.append((st["name"] + " scatter", {k: v for k, v in st.items() if k != "box"}))
    for label, st in variants:
        for adj in (False, True):
            name = st["op"] + ("_adj" if adj else "")
            A, dst = bufs[st["src"]], bufs[st["dst"]]
            launches = []
            if "scatter" in st:
                ptrs = [b.data_ptr() for b in peers[st["dst"]]] if st.get("peer_dst") else [dst.data_ptr()] * P
                for j0, n, spec, p0, pn in pl.parts(st):
                    op = pad_operator(ops[name][2 * j0:2 * (j0 + n)], device=dev)
                    launches.append((op, 2 * n, pl.epi(st, j0, n, spec), ptrs if pn is None else ptrs[p0:p0 + pn]))
            else:
                epi = [0, 0, st["ldc"], 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1, 0]
                launches.append((pad_operator(ops[name], device=dev), st["N"], epi, [dst.data_ptr()]))

            def run():
                for op, N, epi, ptrs in launches:
                    C_.dft_gemm(A, st["M"], st["K"], st["lda"], op, N, epi, ptrs, None, 0, 0)

            ms = time_ms(run, iters, warmup)
            gbs = need[label] / ms / 1e6
            rows.append({"P": P, "Yl": pl.Yl, "staged": pl.staged, "stage": label, "adj": adj,
                         "M": st["M"], "K": st["K"], "N": st["N"], "launches": len(launches), "ms": round(ms, 4),
                         "bytes": need[label], "gbs": round(gbs, 1), "frac_copy": round(gbs / H100_COPY_GBS, 3)})
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ranks", type=int, nargs="+", default=[1, 2, 4, 8])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dft_gemm_bench.py needs a GPU")
    C_ = build.load()
    dev = torch.device("cuda", 0)
    rows = []
    for P in a.ranks:
        for r in cases(C_, P, a.iters, a.warmup, dev):
            rows.append(r)
            print(f"P {P}  Yl {r['Yl']:3d}  {r['stage']:11s} {'adj' if r['adj'] else 'fwd'}  M {r['M']:8d}  K {r['K']:3d}  "
                  f"N {r['N']:3d}  {r['ms']:8.3f} ms  {r['bytes'] / 1e9:6.3f} GB  {r['gbs']:7.1f} GB/s  "
                  f"{r['frac_copy']:5.1%} of copy")
        step = [r for r in rows if r["P"] == P and not r["stage"].endswith(" scatter")]
        print(f"P {P}  all stages, forward + adjoint chain per block x 4 blocks: "
              f"{4 * sum(r['ms'] for r in step):.3f} ms per step")
    state = gpu_state()
    print(f"{state['gpu']}, power limit {state['power_limit_w']} W, SM clock {state['sm_clock_mhz']} MHz "
          f"(max {state['sm_clock_max_mhz']})")
    print(json.dumps({"shape": {"BC": BC, "X": X, "Y": Y, "T": T, "Z": Z, "modes": MODES}, "iters": a.iters,
                      **state, "copy_gbs": H100_COPY_GBS, "cases": rows}))


if __name__ == "__main__":
    main()
