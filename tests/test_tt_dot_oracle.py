"""CPU: the fp64 NumPy chain of tests/ttd_model.py (the computation tnb_tt_dot runs) against the reference's dot, normsq,
norm, dist and relative_error on TT pairs (tests/golden/metrics.npz, written by oracle/gen_metrics.py): fp32 and fp64
cores, different rank profiles, one mode, unit modes, Tucker factors, CP cores and a config-3 pair rebuilt from its
seeds."""
import math
import os

import numpy as np
import pytest

import ttd_model as tm
from oracle import cases

GOLD = os.path.join(os.path.dirname(__file__), "golden", "metrics.npz")


def golden_names():
    g = np.load(GOLD)
    return sorted({k.split("/")[0] for k in g.files if k.endswith("/dot") and not k.startswith("cfg3/")})


def golden_pair(g, name):
    """(a cores, b cores) as plain fp64-or-fp32 TT cores, and the case's dtype."""
    trains = []
    for side in ("a", "b"):
        n = int(g[f"{name}/{side}/n"])
        cores = [g[f"{name}/{side}/core{k}"] for k in range(n)]
        Us = [g[f"{name}/{side}/U{k}"] if f"{name}/{side}/U{k}" in g.files else None for k in range(n)]
        trains.append((cores, Us))
    return trains, trains[0][0][0].dtype


def metrics(a, b):
    """The reference's formulas (metrics.py:119-151, 298-319) on the fp64 chain."""
    ab, aa, bb = tm.dot(a, b), tm.dot(a, a), tm.dot(b, b)
    return dict(dot=ab, normsq_a=aa, norm_a=math.sqrt(max(aa, 0)), norm_b=math.sqrt(max(bb, 0)),
                dist=math.sqrt(aa + bb - 2 * max(ab, 0)), relerr=math.sqrt(max(aa + bb - 2 * ab, 0)) / math.sqrt(max(aa, 0)))


def cfg3_pair(g):
    spec = cases.FULL_ROUND_CASES["cfg3_128x10_r64to16_f64"]
    return cases.make_tt(spec), cases.random_tt(spec["shape"], int(g["cfg3/b_rank"]), int(g["cfg3/b_seed"]))


@pytest.mark.parametrize("name", golden_names())
def test_chain_matches_reference(name):
    g = np.load(GOLD)
    ((ca, Ua), (cb, Ub)), dt = golden_pair(g, name)
    got = metrics(tm.tt_cores(ca, Ua), tm.tt_cores(cb, Ub))
    # the reference computes in the cores' precision: fp32 cases carry its fp32 rounding
    rtol = 2e-5 if dt == np.float32 else 1e-12
    scale = math.sqrt(got["normsq_a"]) * got["norm_b"]  # |<a, b>| can be far below its terms
    for key, v in got.items():
        ref = float(g[f"{name}/{key}"])
        tol = rtol * (scale if key == "dot" else max(abs(ref), got["norm_a"] if key == "normsq_a" else 1.0) *
                      (got["norm_a"] if key == "normsq_a" else 1.0))
        assert abs(v - ref) <= tol, (name, key, v, ref)


def test_config3_chain_matches_reference():
    g = np.load(GOLD)
    a, b = cfg3_pair(g)
    got = metrics(a, b)
    for key, v in got.items():
        ref = float(g[f"cfg3/{key}"])
        tol = 1e-12 * (got["norm_a"] * got["norm_b"] if key == "dot" else abs(ref))
        assert abs(v - ref) <= tol, (key, v, ref)
