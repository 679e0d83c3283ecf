"""Domain-decomposed datasets: every rank reads / generates only its own slab of each sample.

* :class:`DistributedFieldDataset` -- generic ``torch.utils.data.Dataset`` over a *store*
  (anything with ``read(sample, name, slices) -> ndarray``), with global min/max
  normalisation by MIN/MAX all-reduce over the partition and an optional per-rank on-disk
  cache ``{filename}_{sample:04d}_{rank:04d}.npz``.  This is the role of
  reference ``training/two_phase/sleipner_dataset.py:12-121`` (Azure-blob Zarr store,
  HDF5 cache, raw MPI allreduce), generalised: the reference slices only the y axis
  (``:51-55``); here the slab follows the rank's ``P_x`` index on every spatial axis.
* stores: :class:`SyntheticTwoPhaseStore` (procedural CO2-plume-like fields: no network or
  dataset exists in this environment), :class:`NpyDirStore` (``<name>_<i>.npy`` files, memory
  mapped so only the slab is read) and :class:`ZarrStore` (optional ``zarr``/Azure import).
* :func:`generate_batch_indices` -- the helper the reference's Navier-Stokes trainer calls but
  never defines (``experiment_navier_stokes.py:130,157``).
"""
from __future__ import annotations

import os
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist
from torch.utils.data import Dataset

from ..parallel.decomposition import shard_bounds

__all__ = ["DistributedFieldDataset", "DistributedSleipnerDataset3D", "SyntheticTwoPhaseStore", "NpyDirStore",
           "ZarrStore", "generate_batch_indices", "SyntheticNavierStokes"]


def generate_batch_indices(P_x, n: int, batch_size: int, shuffle: bool = True, seed: Optional[int] = None
                           ) -> List[Tuple[int, int]]:
    """``[(a, b), ...]`` batch boundaries over ``n`` samples.  With ``shuffle`` the *order of
    the batches* is drawn on rank 0 and broadcast, so all ranks walk the data identically."""
    bounds = [(a, min(a + batch_size, n)) for a in range(0, n, batch_size)]
    if shuffle:
        order = [None]
        if P_x.rank == 0 or not P_x.active:
            rng = np.random.default_rng(seed)
            order = [rng.permutation(len(bounds)).tolist()]
        if P_x.group is not None and P_x.active:
            dist.broadcast_object_list(order, src=P_x.world_ranks[0], group=P_x.group)
        bounds = [bounds[i] for i in order[0]]
    return bounds


# ------------------------------------------------------------------------------------------ stores
class SyntheticTwoPhaseStore:
    """Deterministic procedural stand-in for the Sleipner CO2 simulations: permeability
    (``permz`` [X,Y,Z]), caprock topography (``tops`` [X,Y]) and a saturation plume
    (``saturation`` [T+1,X,Y,Z]) that spreads from an injection point with time."""

    def __init__(self, shape: Sequence[int], seed: int = 0):
        self.shape = tuple(int(s) for s in shape)          # X, Y, Z, T
        self.seed = seed

    def _coords(self, slices):
        X, Y, Z, _ = self.shape
        ax = [np.arange(n, dtype=np.float32)[s] / n for n, s in zip((X, Y, Z), slices)]
        return np.meshgrid(*ax, indexing="ij")

    def read(self, sample: int, name: str, slices: Tuple[slice, ...]) -> np.ndarray:
        rng = np.random.default_rng(self.seed * 100003 + sample)
        ph = rng.uniform(0, 2 * np.pi, size=6).astype(np.float32)
        cx, cy, cz = rng.uniform(0.3, 0.7, size=3).astype(np.float32)
        T = self.shape[3]
        if name == "tops":
            x, y = np.meshgrid(*[np.arange(n, dtype=np.float32)[s] / n for n, s in zip(self.shape[:2], slices[:2])],
                               indexing="ij")
            return 800 + 30 * np.sin(2 * np.pi * x + ph[0]) * np.cos(2 * np.pi * y + ph[1])
        x, y, z = self._coords(slices[:3] if name != "saturation" else slices[1:4])
        if name == "permz":
            return np.exp(1.5 * np.sin(4 * np.pi * x + ph[2]) * np.sin(2 * np.pi * y + ph[3]) + 0.5 * np.cos(6 * np.pi * z + ph[4]))
        if name == "saturation":
            t = np.arange(T + 1, dtype=np.float32)[slices[0]]
            r2 = (x - cx) ** 2 + (y - cy) ** 2 + 4 * (z - cz) ** 2
            return np.stack([np.clip(0.8 * np.exp(-r2 / (0.002 + 0.01 * ti)) * (ti > 0), 0, 1) for ti in t], 0)
        raise KeyError(name)


class NpyDirStore:
    """``<dir>/<name>_<sample>.npy`` files; memory-mapped so only the requested slab is read."""

    def __init__(self, path: str):
        self.path = path

    def read(self, sample: int, name: str, slices) -> np.ndarray:
        arr = np.load(os.path.join(self.path, f"{name}_{sample}.npy"), mmap_mode="r")
        return np.ascontiguousarray(arr[tuple(slices)])


class ZarrStore:
    """Zarr-backed store (local directory or an Azure blob container client).  ``zarr`` is an
    optional dependency and is not part of this image."""

    def __init__(self, container=None, prefix: str = "", client=None, path: Optional[str] = None):
        try:
            import zarr
        except ImportError as e:                           # pragma: no cover - optional dependency
            raise ImportError("ZarrStore needs the `zarr` package (and azure-storage-blob for blob "
                              "containers); use NpyDirStore or SyntheticTwoPhaseStore otherwise") from e
        self._zarr = zarr
        self.store = zarr.ABSStore(container=container, prefix=prefix, client=client) if client is not None \
            else zarr.DirectoryStore(path)

    def read(self, sample: int, name: str, slices) -> np.ndarray:   # pragma: no cover
        return np.array(self._zarr.core.Array(self.store, path=f"{name}_{sample}")[tuple(slices)])


# ------------------------------------------------------------------------------------------ datasets
class DistributedFieldDataset(Dataset):
    """Two-phase-flow style samples ``x = [permz, tops] -> y = saturation``, layout ``C X Y Z T``.

    ``P_feat`` is the feature partition (``[B, C, X, Y, Z, T]`` grid); ``shape`` the global
    ``(X, Y, Z, T)``."""

    def __init__(self, P_feat, samples, store, shape, normalize: bool = True, savepath: Optional[str] = None,
                 filename: str = "sample", dtype=torch.float32):
        self.P_feat, self.samples, self.store = P_feat, [int(s) for s in samples], store
        self.shape, self.normalize, self.dtype = tuple(int(s) for s in shape), normalize, dtype
        self.savepath, self.filename = savepath, filename
        idx = P_feat.index if P_feat.active else (0,) * P_feat.dim
        grid = [int(g) for g in P_feat.shape[2:5]]
        lo, hi = shard_bounds(self.shape[:3], grid, idx[2:5])
        self.slab = tuple(slice(a, b) for a, b in zip(lo, hi))
        if savepath is not None:
            os.makedirs(savepath, exist_ok=True)

    def __len__(self) -> int:
        return len(self.samples)

    def _cache_file(self, i: int) -> Optional[str]:
        if self.savepath is None:
            return None
        if not self.P_feat.active:      # a rank outside the feature partition owns nothing: no cache file
            return None
        return os.path.join(self.savepath, f"{self.filename}_{i:04d}_{self.P_feat.rank:04d}.npz")

    def _normalise(self, a: np.ndarray) -> np.ndarray:
        """Global min/max scaling to [0, 1] (MIN/MAX all-reduce over the partition)."""
        lo = float(self.P_feat.allreduce_scalar(float(a.min()), "min"))
        a = a - lo
        hi = float(self.P_feat.allreduce_scalar(float(a.max()), "max"))
        return a / hi if hi > 0 else a

    def __getitem__(self, index: int):
        i = self.samples[index]
        cf = self._cache_file(i)
        if cf is not None and os.path.exists(cf):
            z = np.load(cf)
            return torch.from_numpy(z["x"]).to(self.dtype), torch.from_numpy(z["y"]).to(self.dtype)
        sx, sy, sz = self.slab
        T = self.shape[3]
        permz = np.asarray(self.store.read(i, "permz", (sx, sy, sz)), dtype=np.float32)
        tops = np.asarray(self.store.read(i, "tops", (sx, sy)), dtype=np.float32)
        sat = np.asarray(self.store.read(i, "saturation", (slice(0, T + 1), sx, sy, sz)), dtype=np.float32)
        sat = np.clip(np.moveaxis(sat, 0, -1)[..., 1:], 0, None)             # TXYZ -> XYZT, drop t=0
        if self.normalize:
            permz, tops, sat = self._normalise(permz), self._normalise(tops), self._normalise(sat)
        nx, ny, nz = permz.shape
        x = np.stack([permz, np.broadcast_to(tops[:, :, None], (nx, ny, nz))], 0)[..., None]   # C X Y Z 1
        y = sat[None]                                                                         # 1 X Y Z T
        if cf is not None:
            np.savez(cf, x=x, y=y)
        return torch.from_numpy(np.ascontiguousarray(x)).to(self.dtype), torch.from_numpy(np.ascontiguousarray(y)).to(self.dtype)


class DistributedSleipnerDataset3D(DistributedFieldDataset):
    """Name/signature of the reference's dataset class (``sleipner_dataset.py:12-38``); the
    blob-store arguments select a :class:`ZarrStore`, otherwise a synthetic store is used."""

    def __init__(self, P_feat, samples, client=None, container=None, prefix="", shape=(60, 60, 64, 30),
                 normalize=True, padding=None, savepath=None, filename="sleipner", keep_data=False, store=None):
        if store is None:
            store = ZarrStore(container, prefix, client) if client is not None else SyntheticTwoPhaseStore(shape)
        super().__init__(P_feat, samples, store, shape, normalize, savepath, filename)


class SyntheticNavierStokes:
    """Random smooth 2-D vorticity-like trajectories ``u[n, X, Y, T]`` (band-limited noise
    advected in time) standing in for the ``.mat`` file of the reference's NS trainer."""

    @staticmethod
    def make(num: int, n: int, T: int, seed: int = 0) -> torch.Tensor:
        g = torch.Generator().manual_seed(seed)
        kx = torch.fft.fftfreq(n) * n
        k2 = kx[:, None] ** 2 + kx[None, :] ** 2
        amp = torch.exp(-k2 / 18.0)
        w0 = torch.fft.ifft2(amp * torch.fft.fft2(torch.randn(num, n, n, generator=g))).real
        vx, vy = torch.rand(num, generator=g) * 4 - 2, torch.rand(num, generator=g) * 4 - 2
        ts = torch.arange(T, dtype=torch.float32) / T
        ph = torch.exp(-2j * torch.pi * (kx[None, :, None, None] * vx[:, None, None, None] * ts +
                                         kx[None, None, :, None] * vy[:, None, None, None] * ts) / n * 8)
        decay = torch.exp(-0.05 * k2)[None, :, :, None] ** ts
        return torch.fft.ifft2(torch.fft.fft2(w0)[..., None] * ph * decay, dim=(1, 2)).real.float()
