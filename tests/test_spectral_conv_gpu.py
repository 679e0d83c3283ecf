"""The fused engine's spectral convolution, mode by mode, against float64 (H100 only).

Both models get the same weights, with every bypass weight ``blocks.k.linear.W`` set to zero: then the saved
pre-activation of block k is exactly the spectral convolution of the block input ``h_k``, on the fused and on the
legacy pointwise route.  The spectral weights are complex normals of scale 1/sqrt(C), so every retained mode has unit
gain.  One training forward and one backward run on the engine; each block's reference input is the engine's own
saved ``h_k`` (bf16, upcast exactly), which isolates the block from upstream error.  Checks, each at the resolution of
a single Fourier mode:

* forward spectrum: the spectrum entering the channel mix (``_saved["S3"][k]``) against the float64 truncated DFT of
  ``h_k``;
* inverse chain: the float64 ``rfftn`` of the saved pre-activation against the ``rfftn`` of the float64 inverse of
  ``mix(S3, R)`` with the reference model's weights R, at every retained mode (and, on the kt = 0 plane, its mirror:
  the spectrum of a real output is the Hermitian projection there), plus the energy outside those modes;
* adjoint chain: after the backward the pre-activation buffers hold dpre_k, and with W = 0 the engine's input
  gradient of block 0 (``ws["g"]``) is the adjoint spectral convolution of dpre_0 alone.  Both it and every block's
  spectral-weight gradient are compared with the float64 VJP of the portable ``spectral_forward``.

The route matrix reaches every dispatch route ``FusedDistributedFNO`` picks by shape; the two sensitivity tests show
that the checker fails on a single corrupted weight entry and on a single dropped ky column of an operator."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

# Bounds, measured on an H100 80GB HBM3 over seeds 0, 1, 2 and set at about 4x the worst value seen (in brackets).
# Relative Frobenius error and out-of-band energy (energy outside the retained modes over the in-band energy of the
# reference) are at bf16 level on every route:
FRO = {"S3": 1.4e-2, "inverse": 1.8e-2, "adjoint": 2.2e-2, "dR": 5.4e-2}    # [3.35e-3, 4.40e-3, 5.34e-3, 1.35e-2]
OOB = {"inverse": 1.5e-2, "adjoint": 1.6e-2}                                # [3.63e-3, 4.06e-3]
# The per-mode error (see Result) is set by the bf16 rounding of intermediates whose lines are dominated by their zero
# mode, so it grows with the transform lengths and the mean of the field; bounds per configuration,
# (S3, inverse, adjoint, dR) [worst seen]:
MODE = {
    "headline_like": (0.70, 0.90, 0.07, 1.40),        # [0.170, 0.216, 0.0172, 0.332]
    "large_mz": (0.25, 0.66, 0.05, 0.28),             # [0.0612, 0.165, 0.0119, 0.0682]
    "2d_time": (0.10, 0.11, 0.056, 0.30),             # [0.0235, 0.0274, 0.0140, 0.0741]
    "long_t": (0.24, 0.19, 0.045, 0.27),              # [0.0593, 0.0456, 0.0111, 0.0655]
    "long_axes": (0.29, 0.20, 0.042, 0.55),           # [0.0720, 0.0482, 0.0104, 0.137]
    "lift_budget": (0.18, 0.20, 0.035, 0.26),         # [0.0445, 0.0499, 0.00866, 0.0643]
    "resident_operator": (0.25, 0.30, 0.051, 1.00),   # [0.0619, 0.0738, 0.0127, 0.254]
    "small": (0.10, 0.13, 0.04, 0.12),                # [0.0237, 0.0310, 0.00967, 0.0286]
}


def tolerances(case):
    return {kind: dict(mode=m, fro=FRO[kind], oob=OOB.get(kind)) for kind, m in zip(FRO, MODE[case])}


# (id, public in_shape, T, C, modes, expected routes: fused pointwise dataflow, fused front, tensor-core bypass)
ROUTES = [
    ("headline_like", [1, 1, 32, 32, 128, 1], 20, 20, (12, 12, 12, 10), dict(fused_pw=True, front=True, tc=True)),
    ("large_mz", [2, 1, 8, 8, 128, 1], 8, 12, (2, 2, 34, 3), dict(fused_pw=False, front=False, tc=True)),
    ("2d_time", [2, 1, 12, 72, 1], 2, 16, (4, 34, 2), dict(fused_pw=False, front=False, tc=False)),
    ("long_t", [1, 1, 8, 8, 16, 1], 80, 24, (2, 2, 4, 20), dict(fused_pw=True, front=False, tc=True)),
    ("long_axes", [1, 1, 256, 256, 8, 1], 4, 4, (8, 40, 2, 2), dict(fused_pw=True, front=True, tc=True)),
    # the largest configurations on the two envelope boundaries supports() enforces (tests/test_engine_plan.py)
    ("lift_budget", [1, 1, 8, 8, 16, 64], 62, 8, (2, 2, 4, 4), dict(fused_pw=True, front=True, tc=True)),
    ("resident_operator", [1, 1, 4, 256, 8, 1], 4, 4, (2, 48, 2, 2), dict(fused_pw=True, front=True, tc=True)),
]
SMALL = ("small", [1, 1, 16, 16, 16, 1], 8, 8, (4, 4, 4, 3))


# ------------------------------------------------------------------------------------------------ set-up
def _models(in_shape, T, C, modes, blocks=2, seed=0):
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    _, P_x, _ = d.create_standard_partitions([1] * len(in_shape))
    dev = torch.device("cuda")
    torch.manual_seed(seed)
    ref = d.DistributedFNO(P_x, in_shape, T, C, modes, num_blocks=blocks, device=dev, dtype=torch.float64,
                           backend="torch")
    with torch.no_grad():
        for blk in ref.blocks:
            blk.linear.W.zero_()
            for w in blk.weights:
                w.copy_(torch.randn_like(w) / math.sqrt(C))
    fused = FusedDistributedFNO(P_x, in_shape, T, C, modes, num_blocks=blocks, device=dev)
    d.load_global_state(fused, d.gather_global_state(ref, to_all=True), strict=False)
    return d, ref, fused


def _run(fused, in_shape, seed):
    """One training forward and backward; returns the float64 copies the checks need (read before the backward
    overwrites the pre-activations with dpre)."""
    g = torch.Generator(device="cuda").manual_seed(1000 + seed)
    x = torch.randn(*in_shape, device="cuda", generator=g)
    y = fused(x)
    pl = fused.plan
    saved = dict(h=[_pub(h, pl) for h in fused._saved["h"][:pl.num_blocks]],
                 pre=[_pub(p, pl) for p in fused._saved["pre"]],
                 S3=[_spectrum(s, pl) for s in fused._saved["S3"]])
    y.backward(torch.randn(y.shape, device="cuda", generator=g))
    torch.cuda.synchronize()
    saved["dpre"] = [_pub(p, pl) for p in fused._saved["pre"]]
    saved["g"] = _pub(fused.ws["g"], pl)
    saved["dR"] = [_native_weight(fused._seg(f"blocks.{k}.spectral", fused.theta.grad), pl)
                   for k in range(pl.num_blocks)]
    return saved


def _pub(flat, pl):
    """Engine activation [B, C, X, Yl, T, Z] -> float64 [B, C, X, Y, Z, T] (exact)."""
    return flat.view(pl.B, pl.C, pl.X, pl.Yl, pl.T, pl.Z).permute(0, 1, 2, 3, 5, 4).double()


def _spectrum(flat, pl):
    """S3 = [B*C, KZ, mt, KY, KX, (re, im)] -> complex128 [B, C, KZ, mt, KY, KX]: the rows of G3 are (bc, kz, kt, ky),
    its columns (kx, ri) (tests/test_engine_plan.py replays the same layout on the CPU)."""
    return torch.view_as_complex(flat.view(pl.B, pl.C, pl.KZ, pl.mt, pl.KY, pl.KX, 2).double())


def _native_weight(seg, pl):
    """Flat spectral segment [C, C, Q, 2] -> complex128 [i, o, KZ, mt, KY, KX]."""
    return torch.view_as_complex(seg.reshape(pl.C, pl.C, pl.KZ, pl.mt, pl.KY, pl.KX, 2).double())


def _canonical_to_native(w, pl):
    """Canonical [i, o, KX, KY, KZ, mt] (5-D problems: no KX) -> [i, o, KZ, mt, KY, KX]."""
    if w.dim() == 5:
        w = w.unsqueeze(2)
    return w.permute(0, 1, 4, 5, 3, 2)


def _frequencies(pl):
    """DFT index of every retained mode along x, y, z (two-sided) and t (one-sided), in storage order."""
    from dfno_b200.ops.operators import retained_frequencies as rf
    fx = rf(pl.X, pl.mx, True).long() if pl.has_x else torch.zeros(1, dtype=torch.long)
    return fx, rf(pl.Y, pl.my, True).long(), rf(pl.Z, pl.mz, True).long(), torch.arange(pl.mt)


def _grid(pl):
    """Index tensors [KX, KY, KZ, mt] of the retained modes in the rfftn grid [X, Y, Z, T//2 + 1]."""
    return [t.cuda() for t in torch.meshgrid(*_frequencies(pl), indexing="ij")]


def _band(pl):
    """Retained modes of the rfftn grid, plus their mirrors on the planes the rfft keeps both of (kt = 0, T/2)."""
    ix, iy, iz, it = _grid(pl)
    m = torch.zeros(pl.X, pl.Y, pl.Z, pl.T // 2 + 1, dtype=torch.bool, device="cuda")
    m[ix, iy, iz, it] = True
    jt = (-it) % pl.T
    k = jt <= pl.T // 2
    m[((-ix) % pl.X)[k], ((-iy) % pl.Y)[k], ((-iz) % pl.Z)[k], jt[k]] = True
    return m


def _rfftn(v):
    return torch.fft.rfftn(v, dim=(2, 3, 4, 5))


def _truncated_dft(h, pl):
    """float64 truncated DFT of [B, C, X, Y, Z, T] in the S3 order [B, C, KZ, mt, KY, KX]."""
    ix, iy, iz, it = _grid(pl)
    return _rfftn(h)[:, :, ix, iy, iz, it].permute(0, 1, 4, 5, 3, 2)


def _inverse(S4, pl):
    """float64 inverse of a retained spectrum [B, C, KZ, mt, KY, KX]: zero-padded, then irfftn."""
    ix, iy, iz, it = _grid(pl)
    full = torch.zeros(pl.B, pl.C, pl.X, pl.Y, pl.Z, pl.T // 2 + 1, dtype=torch.complex128, device="cuda")
    full[:, :, ix, iy, iz, it] = S4.permute(0, 1, 5, 4, 2, 3)
    return torch.fft.irfftn(full, s=(pl.X, pl.Y, pl.Z, pl.T), dim=(2, 3, 4, 5))


# ------------------------------------------------------------------------------------------------ comparisons
class Result:
    """Entry-by-entry comparison of ``got`` with ``want`` (same shape, complex).

    ``mode``: the largest per-entry error ``|got - want| / (|want| + rms(want))`` and ``worst``, the index of that
    entry: each mode is judged against its own magnitude, with the rms of the reference as the floor.  (A bound on
    ``|err| / rms`` alone would be set by the zero mode: the block inputs are GELU outputs with a mean far above their
    fluctuation, so one bf16-level relative error at the zero mode exceeds the rms of all the other modes.)
    ``fro``: relative Frobenius error; ``oob``: energy outside ``band`` over the in-band energy of ``want``;
    ``flagged``: indices of the entries over ``tol["mode"]``."""

    def __init__(self, name, got, want, tol, band=None):
        err = (got - want).abs()
        w2 = want.abs() ** 2
        if band is not None:
            w2 = w2 * band
            self.oob = float((got.abs() ** 2 * ~band).sum().sqrt() / w2.sum().sqrt())
            err = err * band
            n = int(band.sum()) * (w2.numel() // band.numel())
        else:
            self.oob = None
            n = w2.numel()
        self.name, self.tol = name, tol
        self.rms = float((w2.sum() / n).sqrt())
        self.fro = float(err.norm() / w2.sum().sqrt())
        err = err / (want.abs() + self.rms)
        self.mode = float(err.max())
        self.worst = tuple(int(i) for i in torch.unravel_index(err.argmax(), err.shape))
        flagged = (err > tol["mode"]).nonzero()
        self.n_flagged = flagged.shape[0]
        self.flagged = [tuple(r) for r in flagged[:100000].tolist()]
        self.ok = self.mode <= tol["mode"] and self.fro <= tol["fro"] and (self.oob is None or self.oob <= tol["oob"])

    def metrics(self):
        return dict(mode=self.mode, fro=self.fro, oob=self.oob)

    def __repr__(self):
        return (f"{self.name}: per-mode max {self.mode:.3e} (worst entry {self.worst}), Frobenius {self.fro:.3e}, "
                f"out-of-band {self.oob}, bounds {self.tol}, {self.n_flagged} entries over the per-mode bound")


def check(ref, fused, saved, tol):
    """All per-mode checks of one forward + backward; returns ``{name: Result}``."""
    pl = fused.plan
    band = _band(pl)
    state = {k: v for k, v in _gathered(ref).items() if k.endswith(".spectral")}
    out = {}
    for k in range(pl.num_blocks):
        h = saved["h"][k]
        out[f"S3[{k}]"] = Result(f"S3[{k}]", saved["S3"][k], _truncated_dft(h, pl), tol["S3"])
        R = _canonical_to_native(state[f"blocks.{k}.spectral"], pl).cuda()
        S4 = torch.einsum("biqtyx,ioqtyx->boqtyx", saved["S3"][k], R)
        out[f"inverse[{k}]"] = Result(f"inverse[{k}]", _rfftn(saved["pre"][k]), _rfftn(_inverse(S4, pl)),
                                      tol["inverse"], band)
        # adjoint: float64 VJP of the portable spectral convolution at h_k with cotangent dpre_k
        blk = ref.blocks[k]
        xin = (h.squeeze(2) if fused.five_d else h).clone().requires_grad_()
        dpre = saved["dpre"][k].squeeze(2) if fused.five_d else saved["dpre"][k]
        grads = torch.autograd.grad(blk.spectral_forward(xin), [xin, *blk.weights], dpre)
        gw = torch.zeros(pl.C, pl.C, *blk.fft_shape[2:], dtype=torch.complex128, device="cuda")
        for gr, sl in zip(grads[1:], blk.slices):          # corner blocks -> canonical layout (one rank)
            gw[sl] = gr
        out[f"dR[{k}]"] = Result(f"dR[{k}]", saved["dR"][k], _canonical_to_native(gw, pl), tol["dR"])
        if k == 0:        # ws["g"] holds block 0's input gradient, = spectral^T(dpre_0) because W = 0
            gref = grads[0].unsqueeze(2) if fused.five_d else grads[0]
            out["adjoint[0]"] = Result("adjoint[0]", _rfftn(saved["g"]), _rfftn(gref), tol["adjoint"], band)
    return out


def _gathered(ref):
    import dfno_b200 as d
    return {k: v.cuda() for k, v in d.gather_global_state(ref, to_all=True).items() if k.endswith(".spectral")}


def _routes(fused):
    return dict(fused_pw=fused.fused_pw, front=fused.front is not None, tc=fused.use_tc_bypass)


def measure(case, seed):
    """Metrics of every check for one configuration and seed (how the bounds above were measured)."""
    name, in_shape, T, C, modes = case[:5]
    d, ref, fused = _models(in_shape, T, C, modes, seed=seed)
    res = check(ref, fused, _run(fused, in_shape, seed), tolerances(name))
    return _routes(fused), {k: r.metrics() for k, r in res.items()}


# ------------------------------------------------------------------------------------------------ tests
def test_route_matrix_covers_every_route():
    for flag in ("fused_pw", "front", "tc"):
        assert {r[5][flag] for r in ROUTES} == {True, False}, flag


@pytest.mark.parametrize("case", ROUTES, ids=[r[0] for r in ROUTES])
def test_spectral_convolution_per_mode_matches_float64(case):
    name, in_shape, T, C, modes, routes = case
    d, ref, fused = _models(in_shape, T, C, modes)
    assert _routes(fused) == routes
    res = check(ref, fused, _run(fused, in_shape, 0), tolerances(name))
    for r in res.values():
        print(r)
    bad = [r for r in res.values() if not r.ok]
    assert not bad, bad


@pytest.mark.parametrize("in_shape,nt,width,modes", [
    # 2*KZ > 128: legacy pointwise dataflow (bypass_fwd_tc / bypass_bwd_tc, EPI_HEAD dft_gemm head, head_bwd), B = 2
    ([2, 1, 8, 8, 128, 1], 8, 12, (2, 2, 34, 3)),
    ([2, 1, 12, 72, 1], 2, 16, (4, 34, 2)),                # legacy + CUDA-core bypass and kreduce_gemm (S % 128 = 64)
    ([1, 2, 8, 8, 16, 1], 80, 24, (2, 2, 4, 20)),          # T > 64: z- and t-DFT as two GEMMs instead of spectral_in
], ids=["large_mz", "2d_time", "long_t"])
def test_new_routes_match_the_portable_backend_end_to_end(in_shape, nt, width, modes):
    """The end-to-end check of tests/test_fused_gpu.py (output and every parameter gradient against the fp32 portable
    backend at the reference initialisation) on the routes it has no shape for; it covers the legacy head kernels,
    which the per-mode checks do not reach."""
    import test_fused_gpu as e2e
    e2e.test_forward_backward_match_portable_backend(in_shape, nt, width, modes)


def _perturbed_mode(pl):
    """A retained mode away from kt = 0 (where the Hermitian projection would split an error over two modes):
    (kz, kt, ky, kx) storage indices."""
    return (1, 1, 2, 1 if pl.has_x else 0)


def test_checker_catches_one_corrupted_weight_entry():
    """The engine's copy of one spectral weight (one i, o and mode) is perturbed, the reference keeps the true
    weights: the inverse-chain check fails with that mode as the worst entry; the spectrum entering the mix, which
    comes before the weights, still passes."""
    _, in_shape, T, C, modes = SMALL
    d, ref, fused = _models(in_shape, T, C, modes)
    pl = fused.plan
    saved = _run(fused, in_shape, 0)
    tol = tolerances("small")
    base = check(ref, fused, saved, tol)
    assert all(r.ok for r in base.values()), base
    q = _perturbed_mode(pl)
    S3 = saved["S3"][0]
    fx, fy, fz, ft = _frequencies(pl)
    kz, kt, ky, kx = q
    i = int(S3[(0, slice(None)) + q].abs().argmax())           # the input channel strongest at that mode
    o = 3
    R = _canonical_to_native(_gathered(ref)["blocks.0.spectral"], pl)
    want = _rfftn(_inverse(torch.einsum("biqtyx,ioqtyx->boqtyx", S3, R), pl))[0, o, fx[kx], fy[ky], fz[kz], kt]
    # moves output channel o at that mode by 10x the per-mode bound
    delta = 10 * tol["inverse"]["mode"] * (float(want.abs()) + base["inverse[0]"].rms) / float(S3[0, i][q].abs())
    with torch.no_grad():
        fused._seg("blocks.0.spectral").view(pl.C, pl.C, pl.KZ, pl.mt, pl.KY, pl.KX, 2)[(i, o) + q + (0,)] += delta
    res = check(ref, fused, _run(fused, in_shape, 0), tol)
    print(res)
    assert not res["inverse[0]"].ok
    assert res["inverse[0]"].worst[1:] == (o, int(fx[kx]), int(fy[ky]), int(fz[kz]), kt), res["inverse[0]"]
    assert res["S3[0]"].ok and res["S3[1]"].ok


def test_checker_flags_exactly_the_modes_of_a_dropped_ky_column():
    """Zeroing the (re, im) operator columns of one ky frequency in the forward inverse y-DFT drops that frequency
    from every block output: the inverse-chain check flags modes with that ky (or its mirror on the kt = 0 plane)
    and no other."""
    _, in_shape, T, C, modes = SMALL
    d, ref, fused = _models(in_shape, T, C, modes)
    pl = fused.plan
    j = 1
    with torch.no_grad():
        fused.ops["iG2"][:, 2 * j:2 * j + 2] = 0
    res = check(ref, fused, _run(fused, in_shape, 0), tolerances("small"))
    print(res)
    ky = int(_frequencies(pl)[1][j])
    for k in range(pl.num_blocks):
        r = res[f"inverse[{k}]"]
        assert not r.ok and r.flagged, r
        assert {f[3] for f in r.flagged} <= {ky, (-ky) % pl.Y}, r
    # block 0's input has its full spectrum, so the dropped frequency is flagged away from the kt = 0 plane too
    # (block 1's input inherits the hole there)
    assert any(f[3] == ky and f[5] > 0 for f in res["inverse[0]"].flagged), res["inverse[0]"]
    assert res["S3[0]"].ok
