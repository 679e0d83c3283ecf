#!/usr/bin/env python
"""Record tests/golden/reference_parity.npz: what the UNMODIFIED reference package computes for the cases of
tests/test_reference_parity.py, run on the DistDL / mpi4py stand-in in baseline/compat with the test's seeded
weights (every real or complex floating-point state-dict entry replaced as in ``_seeded_state_dict``).

    oracle/install_reference.sh <path of a slimgroup/dfno checkout>
    python oracle/gen_reference_parity.py

Per rank it stores the reference's state-dict shapes and distribution info, its output, loss (root rank) and the
parameter gradients.  Add a case to CASES here and to the test's parametrisation together.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
COMPAT = os.path.join(ROOT, "baseline", "compat")
sys.path.insert(0, ROOT)
import importlib.util                                          # noqa: E402

from dfno_b200.utils.testing import run_distributed          # noqa: E402

_spec = importlib.util.spec_from_file_location("reference_parity_test",
                                               os.path.join(ROOT, "tests", "test_reference_parity.py"))
_test = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_test)
CFG, _seeded_state_dict = _test.CFG, _test._seeded_state_dict

CASES = [(1, (1, 1, 1, 1, 1, 1)), (4, (1, 1, 2, 2, 1, 1)), (2, (1, 1, 1, 2, 1, 1))]


def _record(rank, ws, grid, in_shape, nt, width, modes, blocks):
    import warnings
    warnings.filterwarnings("ignore")
    for p in (REF, COMPAT):
        if p in sys.path:
            sys.path.remove(p)
    sys.path[:0] = [COMPAT, REF]
    sys.modules.pop("dfno", None)
    import dfno as ref
    assert os.path.abspath(ref.__file__).startswith(REF), ref.__file__
    _, P_ref, _ = ref.create_standard_partitions(grid)
    theirs = ref.DistributedFNO(P_ref, in_shape, nt, width, modes, num_blocks=blocks, dtype=torch.float64)
    sd = theirs.state_dict()
    theirs.load_state_dict(_seeded_state_dict(sd, rank))
    info = ref.compute_distribution_info(P_ref, in_shape)
    xg = torch.randn(*in_shape, dtype=torch.float64, generator=torch.Generator().manual_seed(99))
    y = theirs(xg[tuple(info["slice"])].contiguous())
    t = torch.randn(y.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(5 + rank))
    loss = ref.DistributedRelativeLpLoss(P_ref)(y, t)
    loss.backward()
    out = {"shape": np.array(info["shape"], dtype=np.float64), "start": np.array(info["start"], dtype=np.float64),
           "y": y.detach().numpy(), "loss": np.array([float(loss)]) if rank == 0 else np.zeros(0)}
    for k, v in sd.items():
        out["sdshape/" + k] = np.array(v.shape, dtype=np.float64)
    for k, p in theirs.named_parameters():
        if p.grad is not None:
            out["grad/" + k] = p.grad.detach().numpy()
    return out


def main():
    if not os.path.isdir(os.path.join(REF, "dfno")):
        raise SystemExit("oracle/_ref/dfno is missing: run oracle/install_reference.sh first")
    arrays = {}
    for ws, grid in CASES:
        res = run_distributed(_record, ws, grid, CFG["in_shape"], CFG["nt"], CFG["width"], CFG["modes"], CFG["blocks"],
                              timeout=600)
        for r, d in enumerate(res):
            for k, v in d.items():
                arrays[f"ws{ws}/r{r}/{k}"] = np.asarray(v) if np.iscomplexobj(v) else np.asarray(v, dtype=np.float64)
    out = os.path.join(ROOT, "tests", "golden", "reference_parity.npz")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    np.savez_compressed(out, **arrays)
    print(f"{out}: {len(arrays)} arrays")


if __name__ == "__main__":
    main()
