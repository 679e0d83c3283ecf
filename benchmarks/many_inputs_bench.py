"""Lift kernels and the training step with many input fields (Cin up to 16).

(a) lift_fwd and lift_bwd alone at 128 x 128 x 128, T = 20, for Cin in {1, 4, 5, 8, 16} x Tin in {1, 10} x
    C in {20, 64}, fp32 x, timed with CUDA events over many calls.  Bytes come from the plan's shapes: x + h for the
    forward; dh + x for the backward, + dx (fp32, x's size) when it is formed.  Cin = 4 and 5 sit on either side of
    the dispatch boundary (lift_*_kernel below, lift_*_many_kernel above), so both kernels are measured side by side.
(b) the headline training step (128^3 x 20, width 20, modes 12 12 12 10, 4 blocks) at Cin = 1 and Cin = 16 (Tin = 1),
    alternated in one session, and the Cin = 16 step on the portable fp32 backend (at 64^3 next to the fused one
    when 128^3 does not fit it).

    python benchmarks/many_inputs_bench.py [--iters 20] [--warmup 3]

Prints one line per measurement and one JSON line; writes nothing."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dfno_b200.models.fused import H100_COPY_GBS, EnginePlan  # noqa: E402
from dfno_b200.ops import build  # noqa: E402


def gpu_state():
    """name and power limit (W), read by nvidia-smi in this run"""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, pl = q.stdout.strip().split(", ")
        return {"gpu": name, "power_limit_w": float(pl)}
    except (OSError, ValueError, subprocess.SubprocessError):
        return {"gpu": torch.cuda.get_device_name(), "power_limit_w": None}


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def lift(C_, Cin, Tin, C, iters, warmup):
    """(a): {call: (ms, bytes)}"""
    dev = torch.device("cuda", 0)
    B, X, Y, Z, T = 1, 128, 128, 128, 20
    pl = EnginePlan(B, Cin, Tin, C, T, X, Y, Z, (12, 12, 12, 10))
    pl.finish(4)
    h_bytes = pl.n_act * 2
    x_bytes = B * X * Y * Z * Cin * Tin * 4
    g = torch.Generator(device=dev).manual_seed(100 * Cin + Tin)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)  # noqa: E731
    x = rnd(B, Cin, X, Y, Z, Tin)
    W1, b1, W2, b2 = rnd(T, Tin) / Tin ** 0.5, rnd(T), rnd(C, Cin) / Cin ** 0.5, rnd(C)
    grads = [torch.zeros_like(t) for t in (W1, b1, W2, b2)]
    dims = [B, Cin, Tin, C, T, X, Y, Z]
    h = torch.empty(pl.n_act, device=dev, dtype=torch.bfloat16)
    dh = (rnd(pl.n_act) * 1e-6).to(torch.bfloat16)
    dx = torch.empty_like(x)
    calls = {
        "fwd": (lambda: C_.lift_fwd(x, W1, b1, W2, b2, h, dims), x_bytes + h_bytes),
        "bwd": (lambda: C_.lift_bwd(x, W1, b1, W2, b2, dh, *grads, dims, None), h_bytes + x_bytes),
        "bwd+dx": (lambda: C_.lift_bwd(x, W1, b1, W2, b2, dh, *grads, dims, dx), h_bytes + 2 * x_bytes),
    }
    out = {k: (time_ms(fn, iters, warmup), nb) for k, (fn, nb) in calls.items()}
    del x, h, dh, dx
    torch.cuda.empty_cache()
    return out


def make_step(Cin, backend, n=128):
    """(b): a closure running one training step on n^3 x 20"""
    import dfno_b200 as d
    dev = torch.device("cuda", 0)
    in_shape, T, C, modes = [1, Cin, n, n, n, 1], 20, 20, (12, 12, 12, 10)
    _, P_x, _ = d.create_standard_partitions([1] * 6)
    torch.manual_seed(0)
    fused = backend == "fused"
    net = d.DistributedFNO(P_x, in_shape, T, C, modes, num_blocks=4, device=dev,
                           dtype=torch.bfloat16 if fused else torch.float32, backend=backend)
    assert isinstance(net, d.FusedDistributedFNO) == fused
    opt = d.FusedAdam(net, lr=1e-4) if fused else torch.optim.Adam(net.parameters(), lr=1e-4)
    x = torch.randn(*in_shape, device=dev)

    def one():
        opt.zero_grad()
        net(x).square().sum().backward()
        opt.step()
    return one


def fused_steps(a):
    """(b): the Cin = 1 and Cin = 16 fused steps alternated; {Cin: [ms per window]}"""
    steps = {1: make_step(1, "fused"), 16: make_step(16, "fused")}
    for fn in steps.values():
        time_ms(fn, 1, a.warmup)
    per = {1: [], 16: []}
    for _ in range(a.rounds):
        for cin, fn in steps.items():
            per[cin].append(time_ms(fn, max(3, a.iters // 2), 1))
    return per


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5, help="alternations of the two fused steps")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("many_inputs_bench.py needs a GPU")
    C_ = build.load()
    state = gpu_state()
    res = {**state, "copy_gbs": H100_COPY_GBS, "lift": {}, "step_ms": {}}
    for C in (20, 64):
        for Tin in (1, 10):
            for Cin in (1, 4, 5, 8, 16):
                for k, (ms, nbytes) in lift(C_, Cin, Tin, C, a.iters, a.warmup).items():
                    gbs = nbytes / ms / 1e6
                    kern = "many" if Cin > 4 else "cin<=4"
                    res["lift"][f"{k} C={C} Tin={Tin} Cin={Cin}"] = {
                        "kernel": kern, "ms": round(ms, 4), "gbs": round(gbs, 1), "frac_copy": round(gbs / H100_COPY_GBS, 3)}
                    print(f"lift {k:6s} C={C:2d} Tin={Tin:2d} Cin={Cin:2d} ({kern:6s}) {ms:8.3f} ms {gbs:7.1f} GB/s "
                          f"{gbs / H100_COPY_GBS:6.1%} of copy")
    for cin, v in fused_steps(a).items():
        res["step_ms"][f"fused Cin={cin}"] = round(statistics.median(v), 2)
        print(f"training step, fused, Cin = {cin:2d}: median {statistics.median(v):.2f} ms over {len(v)} windows "
              f"({min(v):.2f} .. {max(v):.2f})")
    torch.cuda.empty_cache()                           # the fused networks are gone with fused_steps' frame
    for n in (128, 64):                                # 64^3: when the portable step does not fit at 128^3
        try:
            ms = round(time_ms(make_step(16, "torch", n), 3, 1), 2)
        except torch.cuda.OutOfMemoryError:
            ms = None                                  # not measured: the shape does not fit this backend
        torch.cuda.empty_cache()
        res["step_ms"][f"portable Cin=16 {n}^3"] = ms
        print(f"training step, portable fp32, Cin = 16, {n}^3: {ms} ms")
        if n == 64:
            ms = round(time_ms(make_step(16, "fused", n), 3, 1), 2)
            torch.cuda.empty_cache()
            res["step_ms"][f"fused Cin=16 {n}^3"] = ms
            print(f"training step, fused, Cin = 16, {n}^3: {ms} ms")
        if ms is not None and n == 128:
            break
    print(f"{state['gpu']}, power limit {state['power_limit_w']} W")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
