"""Golden vectors for tt_multiply (matrix.py:420-443) from the REAL reference, the unmodified package that
oracle/stage_ref.py stages into oracle/_ref/ (`__graft_entry__.build()` stages it where the reference source is present).

    python oracle/gen_matrix.py   ->  tests/golden/tt_multiply.npz

Per case the reference's own cores, the input X and the reference's Y are stored, so tests feed the same cores through
TTMatrix(list_of_cores, ...) and compare the product alone, free of TT-SVD gauge differences."""
import os
import sys
import warnings

import numpy as np

warnings.filterwarnings("ignore")
HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, REPO)

import torch  # noqa: E402

from oracle import stage_ref  # noqa: E402

stage_ref.stage()
tn = stage_ref.load()  # the real reference
if tn is None:
    raise SystemExit("gen_matrix: the reference package is not staged under oracle/_ref")


def random_cores(seed, idims, odims, ranks, dtype):
    g = torch.Generator().manual_seed(seed)
    r = [1] + ranks + [1]
    return [torch.randn(r[k], idims[k], odims[k], r[k + 1], generator=g, dtype=dtype) for k in range(len(idims))]


# name -> (seed, input dims, output dims, inner ranks, X shape, dtype); "ref" is the reference test's own case
CASES = {
    "d1_f64": (11, [7], [5], [], [9, 7], torch.float64),
    "d4_unit_modes_f64": (12, [1, 3, 4, 2], [3, 2, 5, 1], [3, 4, 2], [6, 24], torch.float64),
    "x3d_f64": (13, [3, 4], [2, 5], [6], [4, 5, 12], torch.float64),
    "f32_d2": (14, [4, 6], [5, 3], [8], [17, 24], torch.float32),
    "f32_d3": (15, [2, 3, 2], [3, 2, 4], [4, 5], [64, 12], torch.float32),
}

out = {}
# test_matrix.py::test_tt_multiply at fp64
torch.manual_seed(1)
m = torch.rand(11 * 3, 23 * 2, dtype=torch.float64)
v = torch.rand(30, 11 * 3, dtype=torch.float64)
ttm = tn.TTMatrix(m, input_dims=[11, 3], output_dims=[23, 2], ranks=[50])
specs = {"ref_f64": (ttm.cores, [11, 3], [23, 2], v)}
for name, (seed, idims, odims, ranks, xshape, dtype) in CASES.items():
    cores = random_cores(seed, idims, odims, ranks, dtype)
    X = torch.randn(*xshape, generator=torch.Generator().manual_seed(seed + 100), dtype=dtype)
    specs[name] = (cores, idims, odims, X)
for name, (cores, idims, odims, X) in specs.items():
    t = tn.TTMatrix(list(cores), ranks=[c.shape[-1] for c in cores[:-1]], input_dims=idims, output_dims=odims)
    Y = tn.tt_multiply(t, X)
    out[f"{name}/d"] = np.int64(len(cores))
    for k, c in enumerate(cores):
        out[f"{name}/core{k}"] = c.numpy()
    out[f"{name}/input_dims"] = np.asarray(idims, dtype=np.int64)
    out[f"{name}/output_dims"] = np.asarray(odims, dtype=np.int64)
    out[f"{name}/X"] = X.numpy()
    out[f"{name}/Y"] = Y.numpy()
    print(name, [tuple(c.shape) for c in cores], tuple(X.shape), "->", tuple(Y.shape), Y.dtype, flush=True)

np.savez_compressed(os.path.join(REPO, "tests", "golden", "tt_multiply.npz"), **out)
