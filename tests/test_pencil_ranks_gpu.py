"""Every rank of a 1 x P pencil emulated on one H100, against the float64 portable backend on the whole field.

On one GPU every pointer a kernel would get from CUDA IPC can point at another local buffer, so the engine's multi-rank
code -- peer-scatter epilogues into P ranks' S1 / T1 (direct and staged), the staged permutations, the mix, lift and
head on local shards, the peer-memory all-reduce of the replicated gradients and of the loss sums, and the reassembly
of per-rank shards -- runs here on the module's own code paths.  Three stand-ins make that possible:

* ``_Grid``: the pencil partition of one rank (``fold_onto_pencil`` returns a pencil unchanged, so no Repartition is
  built; ``init_seed`` keeps ``_init_parameters`` from broadcasting).
* ``_Peers.Buffer`` replaces ``SymmetricBuffer``: one allocation per buffer with a guard band on each side (checked
  after every test: a stray peer store would corrupt a neighbouring allocation on a real box) and a payload of bf16 NaN,
  so a slot that no rank wrote shows up as NaN in the output.  The k-th buffer of rank r pairs with the k-th buffer of
  every other rank; ``peer_ptrs()`` resolves the pairing when it is called.
* ``_Peers.Barrier`` replaces ``PeerBarrier``: synchronise the calling thread's stream, then meet the other ranks at a
  ``threading.Barrier``.  The device ``p2p_barrier`` would spin with every peer on one GPU, so it must never launch.

``_Peers.run`` starts one thread per rank, each on its own CUDA stream (the bindings launch on the current stream), so
ranks overlap between barriers and a missing barrier would show up as a race.  The ranks call ``_forward`` /
``_backward`` directly: autograd runs every CUDA node of a device on one worker thread, where the first rank to block in
a barrier would starve the others."""
import threading

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
FWD_TOL, GRAD_TOL = 2e-2, 3e-2
BLOCKS = 2
GUARD = 4096                 # bytes of guard band before and after every emulated symmetric buffer
SENTINEL = 0xA5              # guard byte
BF16_NAN = 0x7FC0            # payload fill (as int16); as fp32 words 0x7FC07FC0 is a NaN too
SPECTRAL_SHARE = 0.3         # least part of the reference output that must come from the spectral path


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


class _Grid:
    """Partition stand-in: rank ``index`` of a 1 x P pencil over the engine's y axis (public Y, or X of a 5-D field)."""

    def __init__(self, nd, P, rank):
        self.dim, self.size = nd, P
        self.shape = [1] * nd
        self.shape[nd - 3] = P
        self.index = [0] * nd
        self.index[nd - 3] = rank
        self.active, self.group, self.world_ranks = True, None, list(range(P))


class _Peers:
    """The ranks of one emulated pencil: symmetric buffers, barrier and the threads that run the ranks."""

    def __init__(self, P):
        self.P = P
        self.bufs = {r: [] for r in range(P)}          # rank -> its buffers in construction order
        self.calls = [0] * P                           # barrier calls per rank
        self.swap = {}                                 # buffer index -> (a, b): its peer_ptrs() swap ranks a and b
        self.gate = threading.Barrier(P, timeout=60)
        peers = self

        class Buffer:
            def __init__(self, nbytes, group=None, rank=0, world=1, device=None):
                assert world == peers.P
                self.nbytes = int((nbytes + 255) // 256 * 256)
                self.rank, self.k = rank, len(peers.bufs[rank])
                peers.bufs[rank].append(self)
                self.mem = torch.empty(self.nbytes + 2 * GUARD, device=DEV, dtype=torch.uint8)
                self.mem[:GUARD].fill_(SENTINEL)
                self.mem[GUARD + self.nbytes:].fill_(SENTINEL)
                self.mem[GUARD:GUARD + self.nbytes].view(torch.int16).fill_(BF16_NAN)
                self.local_ptr = self.mem[GUARD:].data_ptr()

            def view(self, shape, dtype, byte_offset=0):
                n = int(np.prod(shape)) * torch.empty(0, dtype=dtype).element_size()
                assert byte_offset + n <= self.nbytes
                return self.mem[GUARD + byte_offset:GUARD + byte_offset + n].view(dtype).view(list(shape))

            def peer_ptrs(self, byte_offset=0):
                mates = [peers.bufs[p][self.k] for p in range(peers.P)]
                assert all(m.nbytes == self.nbytes for m in mates), "ranks disagree about a buffer's size"
                ptrs = [m.local_ptr + byte_offset for m in mates]
                if self.k in peers.swap:
                    a, b = peers.swap[self.k]
                    ptrs[a], ptrs[b] = ptrs[b], ptrs[a]
                return ptrs

            def close(self):
                pass

        class Barrier:
            def __init__(self, group=None, rank=0, world=1, timeout_s=None):
                self.rank, self.world = rank, world

            def __call__(self):
                if self.world <= 1:
                    return
                peers.calls[self.rank] += 1
                try:
                    torch.cuda.current_stream().synchronize()
                    peers.gate.wait()
                except BaseException:
                    peers.gate.abort()           # the other ranks fail instead of waiting for this one
                    raise

        self.Buffer, self.Barrier = Buffer, Barrier

    def damaged(self):
        """``(rank, k, side)`` of every guard band that no longer holds the sentinel."""
        bad = []
        for r, bufs in self.bufs.items():
            for b in bufs:
                for side, g in (("before", b.mem[:GUARD]), ("after", b.mem[GUARD + b.nbytes:])):
                    if not bool((g == SENTINEL).all()):
                        bad.append((r, b.k, side))
        return bad

    def run(self, fn):
        """``[fn(rank) for rank in range(P)]``, every rank in its own thread on its own stream."""
        self.gate = threading.Barrier(self.P, timeout=60)
        out, errors = [None] * self.P, []

        def body(r):
            try:
                with torch.cuda.device(DEV):
                    s = torch.cuda.Stream()
                    with torch.cuda.stream(s):
                        out[r] = fn(r)
                    s.synchronize()
            except BaseException as e:           # noqa: BLE001 - re-raised in the calling thread
                errors.append(e)
                self.gate.abort()

        threads = [threading.Thread(target=body, args=(r,), name=f"pencil-rank{r}") for r in range(self.P)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if errors:
            first = [e for e in errors if not isinstance(e, threading.BrokenBarrierError)] or errors
            raise first[0]
        return out


@pytest.fixture
def pencil(monkeypatch):
    """``pencil(P, staged)`` -> a fresh :class:`_Peers` installed in place of the peer-memory runtime."""
    from dfno_b200.ops import build
    from dfno_b200.runtime import symm
    mod = build.load()

    def no_device_barrier(*a, **k):
        raise AssertionError("p2p_barrier launched: with every peer on one GPU it would spin")

    monkeypatch.setattr(mod, "p2p_barrier", no_device_barrier)
    made = []

    def make(P, staged=False):
        peers = _Peers(P)
        monkeypatch.setattr(symm, "SymmetricBuffer", peers.Buffer)
        monkeypatch.setattr(symm, "PeerBarrier", peers.Barrier)
        monkeypatch.setenv("DFNO_STAGED_SCATTER", "1" if staged else "0")
        made.append(peers)
        return peers

    yield make
    torch.cuda.synchronize()
    assert not [t for t in threading.enumerate() if t.name.startswith("pencil-rank")]
    for peers in made:
        assert peers.damaged() == [], peers.damaged()


# ------------------------------------------------------------------ cases
class _Case:
    def __init__(self, in_shape, nt, width, modes, padding=None, O=1):
        self.in_shape, self.nt, self.width, self.modes = list(in_shape), nt, width, tuple(modes)
        self.padding, self.O = padding, O
        self.nd = len(in_shape)
        self.out_shape = [in_shape[0], O, *in_shape[2:-1], nt]


CASES = {
    "base": _Case([1, 2, 16, 32, 16, 2], 8, 20, (4, 4, 4, 3)),
    "steady": _Case([1, 1, 16, 32, 16, 1], 1, 20, (4, 4, 4, 1)),
    "padded": _Case([1, 1, 12, 32, 16, 1], 6, 20, (2, 4, 4, 3), padding=(4, 0, 8, 2)),
    "steady_pad_O3": _Case([2, 1, 8, 16, 16, 1], 1, 20, (2, 2, 4, 1), padding=(4, 0, 8, 0), O=3),
    "O4_w24": _Case([1, 1, 16, 16, 16, 1], 8, 24, (4, 4, 4, 3), O=4),
    "cin16_w64": _Case([1, 16, 16, 16, 16, 3], 12, 64, (4, 4, 4, 3)),
    "2d_w48": _Case([2, 1, 32, 32, 10], 16, 48, (4, 4, 4)),
    "long_axes": _Case([1, 1, 256, 256, 8, 1], 4, 4, (8, 40, 2, 2)),
    "long_t": _Case([1, 1, 8, 8, 16, 1], 80, 24, (2, 2, 4, 20)),
    "round1": _Case([2, 1, 8, 8, 128, 1], 8, 12, (2, 2, 34, 3)),
    "round1_cuda_core": _Case([2, 1, 12, 72, 1], 2, 16, (4, 34, 2)),
}

MATRIX = [  # case, P, staged, frozen-weight backward too
    ("base", 2, False, False), ("base", 4, True, False), ("base", 8, True, False), ("base", 8, False, False),
    ("steady", 2, False, False), ("steady", 8, True, False),
    ("padded", 4, False, False),
    ("steady_pad_O3", 2, False, False),
    ("O4_w24", 2, False, False),
    ("cin16_w64", 4, False, True),
    ("2d_w48", 4, True, False),
    ("long_axes", 2, False, False),
    ("long_t", 2, False, False),
    ("round1", 2, False, False), ("round1", 4, False, False),
    ("round1_cuda_core", 2, False, False),
]


class _Reference:
    """The float64 portable backend on the whole field, its output, dL/dx and canonical weight gradients for a
    random output gradient ``dy``, and the canonical state the emulated ranks load.

    The spectral weights are scaled up in steps of 1.4 until the spectral path makes at least ``share`` of the output
    (the relative change when they are zeroed): at the reference initialisation (``U[0,1) / width^2``) it makes well
    under 1 % of it at these shapes, so a broken pencil transpose would pass an output check."""

    def __init__(self, case: _Case, seed=0, blocks=BLOCKS, share=SPECTRAL_SHARE):
        import dfno_b200 as d
        self.case = c = case
        _, P1, _ = d.create_standard_partitions([1] * c.nd)
        torch.manual_seed(seed)
        ref = d.DistributedFNO(P1, c.in_shape, c.nt, c.width, c.modes, num_blocks=blocks, device=DEV,
                               dtype=torch.float64, backend="torch", out_channels=c.O, padding=c.padding)
        g = torch.Generator(device=DEV).manual_seed(seed + 1)
        self.x = torch.randn(*c.in_shape, device=DEV, generator=g)
        self.dy = torch.randn(*c.out_shape, device=DEV, generator=g, dtype=torch.float64)
        self.t = torch.randn(*c.out_shape, device=DEV, generator=g)
        xr = self.x.double().requires_grad_()
        spectral = [w for b in ref.blocks for w in b.weights]
        with torch.no_grad():
            for _ in range(24):
                y = ref(xr)
                saved = [w.detach().clone() for w in spectral]
                for w in spectral:
                    w.zero_()
                self.share = _rel(y, ref(xr))
                for w, s in zip(spectral, saved):
                    w.copy_(s)
                if self.share >= share:
                    break
                for w in spectral:
                    w.mul_(1.4)
        assert self.share >= share, self.share
        self.state = d.gather_global_state(ref, to_all=True)
        self.y = ref(xr)
        self.y.backward(self.dy)
        self.y = self.y.detach()
        self.dx = xr.grad.detach()
        for p in ref.parameters():
            p.data = p.grad if p.grad is not None else torch.zeros_like(p.data)
        self.grads = d.gather_global_state(ref, to_all=True)


def _shards(t, shape, grids):
    from dfno_b200.parallel.decomposition import assemble_slices, shard_bounds
    return [t[assemble_slices(*shard_bounds(shape, g.shape, g.index))].contiguous() for g in grids]


def _engines(c: _Case, P, state=None, init_seed=0, blocks=BLOCKS):
    """The P ranks' engines, built one after another in this thread (the order pairs their symmetric buffers)."""
    from dfno_b200.models.fused import FusedDistributedFNO
    grids = [_Grid(c.nd, P, r) for r in range(P)]
    nets = [FusedDistributedFNO(g, c.in_shape, c.nt, c.width, c.modes, num_blocks=blocks, device=DEV,
                                input_grad=True, out_channels=c.O, padding=c.padding, init_seed=init_seed)
            for g in grids]
    if state is not None:
        for n in nets:
            n.engine_state_from_global(state, strict=False)
    torch.cuda.synchronize()
    return grids, nets


def _canonical(nets, flats):
    """Merged canonical state of the ranks' flat buffers ``flats`` (pointwise entries from rank 0)."""
    parts = [n.theta_to_canonical(f, n.engine_meta(), include_pointwise=n.rank == 0) for n, f in zip(nets, flats)]
    return nets[0].merge_canonical(parts, nets[0].engine_meta())


def _real(t):
    return torch.view_as_real(t) if t.is_complex() else t


@pytest.mark.parametrize("name,P,staged,frozen", MATRIX,
                         ids=[f"{n}-P{P}-{'staged' if s else 'direct'}" for n, P, s, _ in MATRIX])
def test_emulated_ranks_match_float64_backend(pencil, name, P, staged, frozen):
    from dfno_b200.models.fused import FusedAdam
    from dfno_b200.models.loss import _EngineReducedLoss
    c = CASES[name]
    ref = _Reference(c)
    peers = pencil(P, staged)
    grids, nets = _engines(c, P, ref.state)
    pl = nets[0].plan
    assert nets[0].world == P and pl.staged == staged
    xs = _shards(ref.x, c.in_shape, grids)
    dys, ts = _shards(ref.dy, c.out_shape, grids), _shards(ref.t, c.out_shape, grids)
    n_bar = sum(1 for st in nets[0].chain_desc if st.get("barrier_after"))

    def rank(r):
        net, out = nets[r], {}
        n0 = peers.calls[r]
        out["y_eval"] = net._forward(xs[r], save=False)
        n1 = peers.calls[r]
        out["y"] = net._forward(xs[r], save=True)
        n2 = peers.calls[r]
        with torch.no_grad():
            out["rel2"] = _EngineReducedLoss.apply(out["y"], ts[r], net, "rel2").clone()
            out["mse"] = _EngineReducedLoss.apply(out["y"], ts[r], net, "mse").clone()
        n3 = peers.calls[r]
        out["dx"] = net._backward(xs[r], dys[r].float(), input_grad=True, theta_grad=True)
        n4 = peers.calls[r]
        out["grad"] = net.grad_flat.clone()
        if frozen:                     # that backward used up the saved pre-activations: save them again
            grad = net.theta.grad
            net._forward(xs[r], save=True)
            out["dx_frozen"] = net._backward(xs[r], dys[r].float(), input_grad=True, theta_grad=False)
            out["grad_kept"] = net.theta.grad is grad and torch.equal(grad, out["grad"])
        FusedAdam(net, lr=1e-3).step()
        out["small"] = net.theta.data[:pl.n_small].clone()
        out["barriers"] = (n1 - n0, n2 - n1, n3 - n2, n4 - n3)
        return out

    res = peers.run(rank)
    ys_ref, dx_ref = _shards(ref.y, c.out_shape, grids), _shards(ref.dx, c.in_shape, grids)
    print(f"\n{name} P={P} {'staged' if staged else 'direct'}: spectral share of the output {ref.share:.2f}")

    # forward, training and eval buffers: every rank's shard on its own, then the whole field
    for key in ("y", "y_eval"):
        errs = [_rel(o[key], w) for o, w in zip(res, ys_ref)]
        whole = _rel(torch.cat([o[key] for o in res], dim=c.nd - 3), ref.y)
        print(f"  forward ({key}) rel err {whole:.2e}, per rank {['%.1e' % e for e in errs]}")
        assert whole < FWD_TOL and max(errs) < FWD_TOL, (key, whole, errs)

    # loss: the all-reduced sums are bitwise the same on every rank and equal the float64 loss of the engine output
    y_all = torch.cat([o["y"] for o in res], dim=c.nd - 3).double()
    t_all = ref.t.double()
    B = c.in_shape[0]
    want = {"rel2": float(((y_all - t_all).reshape(B, -1).norm(dim=1) / t_all.reshape(B, -1).norm(dim=1)).mean()),
            "mse": float(((y_all - t_all) ** 2).mean())}
    for kind in ("rel2", "mse"):
        vals = [o[kind] for o in res]
        assert all(torch.equal(v, vals[0]) for v in vals), (kind, [float(v) for v in vals])
        got = float(vals[0])
        print(f"  loss {kind} {got:.6e} (float64 of the engine output {want[kind]:.6e})")
        assert abs(got - want[kind]) <= 1e-5 * abs(want[kind]), (kind, got, want[kind])

    # dL/dx
    errs = [_rel(o["dx"].view(w.shape), w) for o, w in zip(res, dx_ref)]
    whole = _rel(torch.cat([o["dx"].view(w.shape) for o, w in zip(res, dx_ref)], dim=c.nd - 3), ref.dx)
    print(f"  dx rel err {whole:.2e}, per rank {['%.1e' % e for e in errs]}")
    assert whole < GRAD_TOL and max(errs) < GRAD_TOL, (whole, errs)
    if frozen:
        for o in res:                  # theta.grad kept; nothing on the dx path is atomic: the same dx bit for bit
            assert o["grad_kept"] and torch.equal(o["dx_frozen"], o["dx"])
        print("  frozen-weight backward: theta.grad kept, dx bitwise equal")

    # weight gradients: the replicated segment bitwise the same everywhere, the merged shards against float64
    for o in res[1:]:
        assert torch.equal(o["grad"][:pl.n_small], res[0]["grad"][:pl.n_small])
    G = _canonical(nets, [o["grad"] for o in res])
    worst = 0.0
    for seg in pl.segments:
        e = _rel(_real(G[seg]).reshape(-1), _real(ref.grads[seg]).reshape(-1))
        worst = max(worst, e)
        assert e < GRAD_TOL, (seg, e)
    print(f"  weight grads: worst segment rel err {worst:.2e}")

    # one Adam step keeps the replicated weights identical
    for o in res[1:]:
        assert torch.equal(o["small"], res[0]["small"])

    # barriers: the same count on every rank, the count the chain descriptors give
    for o in res:
        fwd_eval, fwd, loss, bwd = o["barriers"]
        assert fwd_eval == fwd == n_bar * BLOCKS and loss == 4, o["barriers"]
        assert fwd + bwd == n_bar * BLOCKS * 2 + 2, o["barriers"]
    assert len(set(peers.calls)) == 1, peers.calls
    print(f"  barriers per rank {peers.calls[0]} ({n_bar} per chain)")


@pytest.mark.parametrize("P", [2, 4, 8])
def test_seeded_initialisation_is_partition_independent(pencil, P):
    """``_init_parameters(seed)``: P ranks build the same model as one rank (``bench.py`` checks an N-rank run against
    a 1-rank run on that promise)."""
    import dfno_b200 as d
    from dfno_b200.models.fused import FusedDistributedFNO
    c = CASES["base"]
    _, P1, _ = d.create_standard_partitions([1] * c.nd)
    one = FusedDistributedFNO(P1, c.in_shape, c.nt, c.width, c.modes, num_blocks=BLOCKS, device=DEV, init_seed=7)
    peers = pencil(P, P >= 8)
    grids, nets = _engines(c, P, init_seed=7)
    mine, want = _canonical(nets, [n.theta.data for n in nets]), _canonical([one], [one.theta.data])
    assert sorted(mine) == sorted(want)
    for k in want:
        assert torch.equal(mine[k], want[k]), k
    x = torch.randn(*c.in_shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    y1 = one._forward(x, save=False)
    xs = _shards(x, c.in_shape, grids)
    yP = torch.cat(peers.run(lambda r: nets[r]._forward(xs[r], save=False)), dim=c.nd - 3)
    print(f"\nP={P}: {P}-rank and 1-rank forwards of the seeded model differ by {_rel(yP, y1):.2e} (relative)")
    assert _rel(yP, y1) < FWD_TOL


def test_swapped_peer_pointers_fail_the_per_rank_check(pencil):
    """The harness can fail: with rank 0's and rank 1's T1 swapped in every rank's peer table, iG2 delivers each of
    the two the other's y slab.  Their shards must then miss by at least 10x the tolerance; the other ranks' must
    not.  One block, so that no later block spreads the two wrong shards over the field."""
    c, P = CASES["base"], 4
    ref = _Reference(c, blocks=1, share=0.6)
    peers = pencil(P)
    grids, nets = _engines(c, P, ref.state, blocks=1)
    k_T1 = 1                                   # construction order: S1, T1, the small all-reduce buffer
    assert peers.bufs[0][k_T1].nbytes == (nets[0].plan.n_T1 * 2 + 255) // 256 * 256
    peers.swap = {k_T1: (0, 1)}
    xs = _shards(ref.x, c.in_shape, grids)
    ys = peers.run(lambda r: nets[r]._forward(xs[r], save=False))
    errs = [_rel(y, w) for y, w in zip(ys, _shards(ref.y, c.out_shape, grids))]
    print(f"\nper-rank forward rel err with T1 of ranks 0 and 1 swapped: {['%.2e' % e for e in errs]}")
    assert min(errs[:2]) > 10 * FWD_TOL, errs
    assert max(errs[2:]) < FWD_TOL, errs


def test_guard_band_check_sees_an_overwritten_sentinel(pencil):
    peers = pencil(2)
    a, b = peers.Buffer(1000, None, 0, 2), peers.Buffer(1000, None, 1, 2)
    assert a.nbytes == b.nbytes == 1024 and a.peer_ptrs() == [a.local_ptr, b.local_ptr] == b.peer_ptrs()
    assert torch.isnan(a.view([512], torch.bfloat16)).all() and torch.isnan(a.view([256], torch.float32)).all()
    assert peers.damaged() == []
    for at, side in ((GUARD + b.nbytes + 17, "after"), (GUARD - 1, "before")):
        b.mem[at] = 0                          # one byte written from the host into the guard band
        assert peers.damaged() == [(1, 0, side)]
        b.mem[at] = SENTINEL
    assert peers.damaged() == []
