"""The TT-cross oracle (tests/cross_model.py) against the reference's own runs: no GPU needed.

`cross.npz` holds tn.cross runs of the reference from seeded global RNGs; `cross_batch.npz` holds B sequential runs of it
from one seed.  The oracle makes the same RNG draws, so it must reproduce their ranks, sample counts and index sets
exactly, and their validation errors to 1e-9 relative.  The oracle's maxvol and rect_maxvol margin restatements are
checked here against py_maxvol / py_rect_maxvol, whose choices they must follow wherever their margins exceed MARGIN.

Two of the reference's runs cannot be reproduced index for index by any implementation that does not round exactly like
the LAPACK build that made them: `cfg5_32x6_r10` and `adaptive_32x5` sample 1 / (shift + sum x), whose sample matrices
are numerically rank deficient at their ranks (sigma_min / sigma_max ~ 1e-16).  The trailing columns of Q are then
rounding noise and the pivots chosen among them are ties.  The test asserts both premises: their smallest
sigma_min / sigma_max is below 1e-12 and their smallest margin below MARGIN.
For those, ranks and sample counts are exact and the validation error, itself at the rounding level of the
interpolation, is compared within 10x."""
import os

import numpy as np
import pytest
import torch

import cross_model as cm
from oracle import cases
from oracle import tt_oracle as orc

GOLD = os.path.join(os.path.dirname(__file__), "golden")
MARGIN = 1e-9
RANK_DEFICIENT = {"cfg5_32x6_r10", "adaptive_32x5"}


def _domain(spec):
    return [np.linspace(spec["lo"], spec["hi"], spec["I"]) for _ in range(spec["N"])]


@pytest.mark.parametrize("name", list(cases.CROSS_CASES))
def test_oracle_reproduces_reference_cross(name):
    g = np.load(os.path.join(GOLD, "cross.npz"))
    spec = cases.CROSS_CASES[name]
    np.random.seed(spec["seed"])
    torch.manual_seed(spec["seed"])
    kw = {k: spec[k] for k in ("ranks_tt", "kickrank", "eps", "max_iter") if k in spec}
    prob = cm.Problem(cases.cross_function(spec.get("shift", 0.0), spec.get("fn")), domain=_domain(spec),
                      minimize=bool(spec.get("minimize")))
    cores, info = cm.run(prob, **kw)
    print(f"{name}: smallest margin {info['margin']:.2e} over {info['steps']} steps")
    assert list(info["Rs"]) == list(g[f"{name}/Rs"])
    assert info["nsamples"] == int(g[f"{name}/nsamples"])
    ref = float(g[f"{name}/val_eps"])
    if name in RANK_DEFICIENT:
        assert info["margin"] < MARGIN and info["cond"] < 1e-12, (info["margin"], info["cond"])
        assert ref / 10 <= info["val_eps"] <= 10 * ref, (info["val_eps"], ref)
        return
    assert np.array_equal(info["lsets"][-1], g[f"{name}/lset_last"])
    if spec.get("minimize"):
        assert abs(float(info["min"]) - float(g[f"{name}/min"])) <= 1e-12
        assert info["argmin"] == tuple(int(v) for v in g[f"{name}/argmin"])
    assert abs(info["val_eps"] - ref) <= 1e-9 * ref, (info["val_eps"], ref)


@pytest.mark.parametrize("name", list(cases.CROSS_BATCH_CASES))
def test_oracle_reproduces_reference_cross_batch(name):
    g = np.load(os.path.join(GOLD, "cross_batch.npz"))
    spec = cases.CROSS_BATCH_CASES[name]
    np.random.seed(spec["seed"])
    torch.manual_seed(spec["seed"])
    probs = [cm.Problem(cases.cross_family_function(b, spec["family"]), domain=_domain(spec))
             for b in range(spec["nproblems"])]
    runs = cm.run_batch(probs, spec["ranks_tt"], eps=spec.get("eps", 1e-6), max_iter=spec["max_iter"])
    assert [i["nsamples"] for _, i in runs] == list(g[f"{name}/nsamples"])
    assert [len(i["val_epss"]) for _, i in runs] == list(g[f"{name}/iters"])
    probe = np.stack([cm.tt_values(c, g[f"{name}/probe_idx"]) for c, _ in runs])
    np.testing.assert_allclose(probe, g[f"{name}/probe"], rtol=1e-9, atol=0)
    # the family is rank deficient like cfg5_32x6_r10 (see the module docstring): its validation errors are rounding noise
    ve = np.array([i["val_eps"] for _, i in runs])
    assert np.all(ve <= np.maximum(10 * g[f"{name}/val_eps"], 1e-11)), (ve, g[f"{name}/val_eps"])


@pytest.mark.parametrize("name", list(cases.MAXVOL_CASES))
def test_maxvol_margins_agree_with_py_maxvol(name):
    """The margin restatement follows py_maxvol's decisions on the reference's maxvol goldens."""
    g = np.load(os.path.join(GOLD, "maxvol.npz"))
    A = cases.make_matrix(cases.MAXVOL_CASES[name])
    idx, C, info = cm.maxvol(A)
    assert list(idx) == list(g[f"{name}/index"])
    if A.shape[0] > A.shape[1]:
        assert info["margin"] > MARGIN and len(info["lu"]) == A.shape[1]


def test_maxvol_margin_sees_exact_ties():
    rng = np.random.default_rng(0)
    A = rng.standard_normal((40, 4))
    top = int(np.argmax(np.abs(A[:, 0])))
    A[39] = -A[top]
    idx, _, info = cm.maxvol(A)
    assert info["lu"][0] == 0.0 and info["margin"] == 0.0
    assert idx[0] != 39  # the lower row wins the tie (LAPACK idamax)


def test_maxvol_swap_count_and_stopping_rules():
    rng = np.random.default_rng(1)
    A = rng.standard_normal((300, 6))
    idx, C, info = cm.maxvol(A)
    assert info["iters"] > 0
    idx0, _, info0 = cm.maxvol(A, max_iters=0)
    assert info0["iters"] == 0 and list(idx0) == list(cm._lu_pivots(A)[0])
    assert list(cm.maxvol(A, tol=0.5)[0]) == list(cm.maxvol(A, tol=1.0)[0])


@pytest.mark.parametrize("kw", [dict(tol=1.0), dict(tol=0.5, maxK=15), dict(tol=2.0, minK=12), dict(min_add_K=3, maxK=20)])
def test_rect_maxvol_margins_agree_with_py_rect_maxvol(kw):
    A = np.random.default_rng(2).standard_normal((200, 8))
    idx, C, info = cm.rect_maxvol(A, **kw)
    ri, rC = orc.py_rect_maxvol(A, **kw)
    assert list(idx) == list(ri) and np.array_equal(C, rC)
    assert len(info["add"]) == len(idx) - 8


def test_fibres_order_matches_reshape():
    lset = np.array([[0, 3, 1], [0, 2, 2]])
    rset = np.array([[4, 0], [1, 0], [0, 0]])
    M = cm.fibres(lset, rset, 5)
    assert M.shape == (2 * 5 * 3, 4)
    a, i, c = 1, 3, 2
    assert list(M[(a * 5 + i) * 3 + c]) == [2, 2, 3, 0]


def test_tensors_input_equals_grid_input():
    """Sampling through input TTs (cross(tensors=...)) equals indexing the grid when the TTs are the meshgrid."""
    rng = np.random.default_rng(3)
    axes = [rng.standard_normal(n) for n in (4, 5, 6)]
    mesh = []
    for k in range(3):
        mesh.append([axes[n].reshape(1, -1, 1) if n == k else np.ones((1, len(axes[n]), 1)) for n in range(3)])
    M = np.stack([rng.integers(0, n, 30) for n in (4, 5, 6)], axis=1)
    a = cm.Problem(lambda *x: x[0], domain=axes).coords(M)
    b = cm.Problem(lambda *x: x[0], tensors=mesh).coords(M)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
