"""Golden vectors for the rounded elementwise product from the REAL reference, the unmodified package that
oracle/stage_ref.py stages into oracle/_ref/.

    python oracle/gen_hadamard_round.py   ->  tests/golden/hadamard_round.npz

Per case: the operands' TT cores (CP and TT-Tucker operands already converted by the reference's own
decompress_tucker_factors / _cp_to_tt, so the cores are what both packages multiply), eps, rmax, and the reference's
tn.round_tt(t1 * t2) ranks and relative error to the exact product.  'reduce/*' cases store tn.reduce([...], operator.mul)
and 'hsum/*' cases tn.hadamard_sum(..., 'svd', eps) with the exact sum."""
import operator
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
    raise SystemExit("gen_hadamard_round: the reference package is not staged under oracle/_ref")


def tt(seed, shape, ranks, dtype):
    g = torch.Generator().manual_seed(seed)
    r = [1] + ranks + [1]
    return tn.Tensor([torch.randn(r[k], shape[k], r[k + 1], generator=g, dtype=dtype) for k in range(len(shape))])


def as_tt(t):
    t = t.decompress_tucker_factors()
    t._cp_to_tt()
    return t


def tucker(seed, shape, ranks, dtype):
    g = torch.Generator().manual_seed(seed)
    r = [1] + ranks + [1]
    S = [max(2, s - 1) for s in shape]
    cores = [torch.randn(r[k], S[k], r[k + 1], generator=g, dtype=dtype) for k in range(len(shape))]
    Us = [torch.randn(shape[k], S[k], generator=g, dtype=dtype) for k in range(len(shape))]
    return tn.Tensor(cores, Us=Us)


def cp(seed, shape, R, dtype):
    g = torch.Generator().manual_seed(seed)
    return tn.Tensor([torch.randn(s, R, generator=g, dtype=dtype) for s in shape])


F32, F64 = torch.float32, torch.float64
CASES = {
    # name: (t1, t2, eps, rmax)
    "r_small_f64": (lambda: tt(1, [6, 5, 7, 4], [3, 4, 3], F64), lambda: tt(2, [6, 5, 7, 4], [4, 2, 3], F64), 1e-6, 0),
    "r_small_f32": (lambda: tt(3, [6, 5, 7, 4], [3, 4, 3], F32), lambda: tt(4, [6, 5, 7, 4], [4, 2, 3], F32), 1e-3, 0),
    "r_rmax_f64": (lambda: tt(5, [8, 8, 8, 8], [5, 6, 5], F64), lambda: tt(6, [8, 8, 8, 8], [4, 5, 4], F64), 0.0, 6),
    "r576_f64": (lambda: tt(7, [4] * 6, [24] * 5, F64), lambda: tt(8, [4] * 6, [24] * 5, F64), 1e-2, 0),
    "r576_f32": (lambda: tt(9, [4] * 6, [24] * 5, F32), lambda: tt(10, [4] * 6, [24] * 5, F32), 1e-2, 0),
    "r576_rmax_f64": (lambda: tt(11, [8] * 6, [24] * 5, F64), lambda: tt(12, [8] * 6, [24] * 5, F64), 0.0, 20),
    "tucker_cp_f64": (lambda: tucker(13, [6, 7, 5, 6], [3, 4, 3], F64), lambda: cp(14, [6, 7, 5, 6], 4, F64), 1e-8, 0),
    "n1_f64": (lambda: tt(15, [9], [], F64), lambda: tt(16, [9], [], F64), 1e-14, 0),
    "n2_f32": (lambda: tt(17, [7, 9], [5], F32), lambda: tt(18, [7, 9], [4], F32), 1e-4, 0),
    "zero_f32": (lambda: tt(19, [5, 6, 4], [3, 2], F32), lambda: tn.Tensor([c * 0 for c in tt(20, [5, 6, 4], [2, 3], F32).cores]),
                 1e-10, 0),
}


def main():
    out = {}
    for name, (f1, f2, eps, rmax) in CASES.items():
        t1, t2 = as_tt(f1()), as_tt(f2())
        N = t1.dim()
        exact = (t1 * t2)
        r = tn.round_tt(exact, eps=eps, rmax=rmax if rmax > 0 else np.iinfo(np.int32).max)
        full, approx = exact.torch().double(), r.torch().double()
        nrm = torch.norm(full)
        err = float(torch.norm(full - approx) / nrm) if nrm > 0 else 0.0
        out[f"{name}/N"] = np.array(N)
        out[f"{name}/eps"] = np.array(eps)
        out[f"{name}/rmax"] = np.array(rmax)
        for k in range(N):
            out[f"{name}/a{k}"] = t1.cores[k].numpy()
            out[f"{name}/b{k}"] = t2.cores[k].numpy()
        out[f"{name}/ranks"] = np.array([int(x) for x in r.ranks_tt])
        out[f"{name}/relerr"] = np.array(err)
        print(name, [int(x) for x in r.ranks_tt], err)
    # tn.reduce over four operands of ranks 4: the first level's products have rank 16, the second level's 36^2
    for dt, tag in ((F64, "f64"), (F32, "f32")):
        ts = [tt(30 + k, [6] * 5, [4] * 4, dt) for k in range(4)]
        r = tn.reduce(ts, operator.mul, eps=1e-3)
        full = ts[0].torch().double() * ts[1].torch().double() * ts[2].torch().double() * ts[3].torch().double()
        err = float(torch.norm(full - r.torch().double()) / torch.norm(full))
        for i, t in enumerate(ts):
            for k in range(5):
                out[f"reduce_{tag}/t{i}_{k}"] = t.cores[k].numpy()
        out[f"reduce_{tag}/ranks"] = np.array([int(x) for x in r.ranks_tt])
        out[f"reduce_{tag}/relerr"] = np.array(err)
        print("reduce", tag, [int(x) for x in r.ranks_tt], err)
    # hadamard_sum with the approximate algorithm, against the exact sum (the reference's builds float32 cores)
    for dt, tag in ((F32, "f32"),):
        ts = [tt(40 + k, [5] * 4, [3] * 3, dt) for k in range(3)]
        approx = tn.hadamard_sum(ts, algorithm="svd", eps=1e-6)
        exact = tn.hadamard_sum(ts, algorithm="exact")
        for i, t in enumerate(ts):
            for k in range(4):
                out[f"hsum_{tag}/t{i}_{k}"] = t.cores[k].numpy()
        out[f"hsum_{tag}/svd"] = np.array(float(approx))
        out[f"hsum_{tag}/exact"] = np.array(float(exact))
        print("hsum", tag, approx, exact)
    np.savez_compressed(os.path.join(REPO, "tests", "golden", "hadamard_round.npz"), **out)


if __name__ == "__main__":
    main()
