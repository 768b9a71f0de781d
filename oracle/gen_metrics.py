"""Golden vectors for the inner-product metrics (metrics.py:28-151, 298-319) from the REAL reference, the unmodified
package that oracle/stage_ref.py stages into oracle/_ref/.

    python oracle/gen_metrics.py   ->  tests/golden/metrics.npz

Per case the operands' cores (and Tucker factors) and the reference's dot, normsq, norm, dist and relative_error on the
pair are stored.  The config-3 pair (128^10, ranks 64 and 16, fp64) stores only its results: its cores are rebuilt from
the seeds in oracle/cases.py, as full.npz's are."""
import os
import sys
import warnings

import numpy as np

warnings.filterwarnings("ignore")
HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, REPO)

import torch  # noqa: E402

from oracle import cases, stage_ref  # noqa: E402

stage_ref.stage()
tn = stage_ref.load()  # the real reference
if tn is None:
    raise SystemExit("gen_metrics: the reference package is not staged under oracle/_ref")


def tt(seed, shape, ranks, dtype):
    g = torch.Generator().manual_seed(seed)
    r = [1] + ranks + [1]
    return [torch.randn(r[k], shape[k], r[k + 1], generator=g, dtype=dtype) for k in range(len(shape))]


def factors(seed, shape, sizes, dtype):
    """Tucker factors [I, S] on the modes where sizes[k] is not None."""
    g = torch.Generator().manual_seed(seed)
    return [None if s is None else torch.randn(shape[k], s, generator=g, dtype=dtype) for k, s in enumerate(sizes)]


def cp(seed, shape, R, dtype):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, R, generator=g, dtype=dtype) for n in shape]


f64, f32 = torch.float64, torch.float32
S4 = [4, 5, 6, 3]
# name -> (a cores, a Us, b cores, b Us); every pair has one shape
CASES = {
    "f64_ranks": (tt(1, S4, [3, 4, 2], f64), None, tt(2, S4, [2, 5, 3], f64), None),
    "f32_ranks": (tt(3, S4, [3, 4, 2], f32), None, tt(4, S4, [2, 5, 3], f32), None),
    "f64_one_mode": (tt(5, [9], [], f64), None, tt(6, [9], [], f64), None),
    "f64_unit_modes": (tt(7, [1, 3, 1, 4, 1], [2, 3, 3, 2], f64), None, tt(8, [1, 3, 1, 4, 1], [1, 2, 4, 1], f64), None),
    "f64_tc_ranks": (tt(9, [6, 5, 7, 4], [16, 24, 20], f64), None, tt(10, [6, 5, 7, 4], [20, 16, 32], f64), None),
    "f32_tc_ranks": (tt(11, [6, 5, 7, 4], [16, 24, 20], f32), None, tt(12, [6, 5, 7, 4], [20, 16, 32], f32), None),
    "f64_tucker": (tt(13, [3, 5, 2, 5], [2, 3, 2], f64), factors(14, S4, [3, None, 2, 5], f64),
                   tt(15, S4, [3, 2, 2], f64), None),
    "f64_cp": (cp(16, S4, 3, f64), None, tt(17, S4, [2, 3, 2], f64), None),
    "f32_cp_tucker": (cp(18, [2, 5, 3, 3], 4, f32), factors(19, S4, [2, None, 3, None], f32),
                      tt(20, S4, [3, 3, 2], f32), factors(21, S4, [None] * 4, f32)),
}

out = {}
for name, (ca, Ua, cb, Ub) in CASES.items():
    a, b = tn.Tensor(list(ca), Us=Ua), tn.Tensor(list(cb), Us=Ub)
    res = dict(dot=tn.dot(a, b), normsq_a=tn.normsq(a), norm_a=tn.norm(a), norm_b=tn.norm(b), dist=tn.dist(a, b),
               relerr=tn.relative_error(a, b))
    for side, cs, Us in (("a", ca, Ua), ("b", cb, Ub)):
        out[f"{name}/{side}/n"] = np.int64(len(cs))
        for k, c in enumerate(cs):
            out[f"{name}/{side}/core{k}"] = c.numpy()
            if Us is not None and Us[k] is not None:
                out[f"{name}/{side}/U{k}"] = Us[k].numpy()
    for key, v in res.items():
        out[f"{name}/{key}"] = np.float64(float(v))
    print(name, {k: float(v) for k, v in res.items()}, flush=True)

# config 3: tn.randn([128]*10, ranks_tt=64) against a rank-16 train of the same shape, fp64
spec = cases.FULL_ROUND_CASES["cfg3_128x10_r64to16_f64"]
a = tn.Tensor([torch.from_numpy(c) for c in cases.make_tt(spec)])
B_SEED = 125
b = tn.Tensor([torch.from_numpy(c) for c in cases.random_tt(spec["shape"], 16, B_SEED)])
res = dict(dot=tn.dot(a, b), normsq_a=tn.normsq(a), norm_a=tn.norm(a), norm_b=tn.norm(b), dist=tn.dist(a, b),
           relerr=tn.relative_error(a, b))
out["cfg3/b_seed"] = np.int64(B_SEED)
out["cfg3/b_rank"] = np.int64(16)
for key, v in res.items():
    out[f"cfg3/{key}"] = np.float64(float(v))
print("cfg3", {k: float(v) for k, v in res.items()}, flush=True)

np.savez_compressed(os.path.join(REPO, "tests", "golden", "metrics.npz"), **out)
