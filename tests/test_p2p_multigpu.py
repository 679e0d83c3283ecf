"""Peer-memory data plane on several H100s: push all-to-all-v vs NCCL, Repartition over it
(values + adjoint), flag barrier and small all-reduce."""
import numpy as np
import pytest
import torch

from dfno_b200.utils.testing import run_distributed

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def _a2a(rank, ws):
    import torch.distributed as dist
    from dfno_b200.runtime.symm import P2PAllToAll, PeerBarrier, SymmetricBuffer
    from dfno_b200.ops import build
    dev = torch.device("cuda", torch.cuda.current_device())
    eng = P2PAllToAll(dist.group.WORLD, rank, ws, 1 << 22)
    g = torch.Generator(device=dev).manual_seed(rank)
    for trial, dtype in enumerate([torch.bfloat16, torch.float32, torch.float32]):
        # uneven, non-16-byte-multiple segment sizes
        counts = [[(7 + 13 * s + 5 * d_ + 3 * trial) % 23 * (64 if trial < 2 else 1) + 1 for s in range(ws)]
                  for d_ in range(ws)]                       # counts[d][s]: s -> d
        send_counts = [counts[d_][rank] for d_ in range(ws)]
        send = torch.randn(sum(send_counts), device=dev, generator=g).to(dtype)
        got = eng.exchange(send, send_counts, counts)
        want = torch.empty(sum(counts[rank]), device=dev, dtype=dtype)
        dist.all_to_all_single(want, send, counts[rank], send_counts)
        assert torch.equal(got, want)
    # small all-reduce through peer reads
    bar = PeerBarrier(dist.group.WORLD, rank, ws)
    buf = SymmetricBuffer(4096, dist.group.WORLD, rank, ws)
    mine = torch.arange(1000, device=dev, dtype=torch.float32) * (rank + 1)
    buf.view([1000], torch.float32).copy_(mine)
    bar()
    out = torch.empty(1000, device=dev)
    build.load().p2p_allreduce_small(buf.peer_ptrs(), out, 1000, rank)
    bar()
    assert torch.equal(out, torch.arange(1000, device=dev, dtype=torch.float32) * sum(range(1, ws + 1)))
    torch.cuda.synchronize()
    return True


def _repart(rank, ws, grid_a, grid_b, shape, cplx):
    import dfno_b200 as d
    from dfno_b200.parallel.decomposition import shard_bounds, assemble_slices
    from dfno_b200.parallel import primitives
    dev = torch.device("cuda", torch.cuda.current_device())
    P_w = d.Partition()
    Pa = P_w.create_partition_inclusive(range(int(np.prod(grid_a)))).create_cartesian_topology_partition(grid_a)
    Pb = P_w.create_partition_inclusive(range(int(np.prod(grid_b)))).create_cartesian_topology_partition(grid_b)
    dt = torch.complex64 if cplx else torch.float32
    torch.manual_seed(1)
    G, H = torch.randn(*shape, dtype=dt), torch.randn(*shape, dtype=dt)

    def shard(P, T):
        if not P.active:
            return d.zero_volume_tensor(dtype=dt, device=dev)
        lo, hi = shard_bounds(shape, P.shape, P.index)
        return T[assemble_slices(lo, hi)].clone().to(dev)

    R = d.Repartition(Pa, Pb, shape, dtype=dt)
    x = shard(Pa, G).requires_grad_()
    y = R(x)
    assert torch.equal(y.detach(), shard(Pb, G))
    y.backward(shard(Pb, H))
    assert torch.equal(x.grad, shard(Pa, H))
    assert len(primitives._P2P_POOL) == 1, "the peer-memory engine was not used"
    torch.cuda.synchronize()
    return True


def test_p2p_alltoall_barrier_allreduce():
    import os
    n = 4 if torch.cuda.device_count() >= 4 and os.environ.get("DFNO_TEST_WORLD", "2") == "4" else 2
    assert all(run_distributed(_a2a, n, cuda=True, timeout=300))


@pytest.mark.parametrize("grid_a,grid_b,shape,cplx", [
    ((1, 1, 1, 2), (1, 1, 2, 1), (2, 3, 10, 9), False),
    ((1, 1, 2, 1), (1, 1, 1, 2), (1, 4, 7, 12), True),
])
def test_repartition_over_peer_memory(grid_a, grid_b, shape, cplx):
    assert all(run_distributed(_repart, 2, grid_a, grid_b, shape, cplx, cuda=True, timeout=300))
