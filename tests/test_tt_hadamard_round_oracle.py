"""CPU: the Gram-form rounding of an elementwise product (tests/tthr_model.py, the method of tnb_tt_hadamard_round)
against the fp64 oracle's round_tt on the explicit Kronecker cores, and against the reference's own results."""
import os

import numpy as np
import pytest

import tthr_model as hm
from oracle import tt_oracle as orc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hadamard_round.npz")


def _tt(rng, shape, ranks):
    r = [1] + list(ranks) + [1]
    return [rng.standard_normal((r[k], shape[k], r[k + 1])) for k in range(len(shape))]


CASES = [
    # (shape, ranks a, ranks b, eps, rmax)
    ([5, 6, 4, 5], [3, 4, 2], [2, 3, 3], 1e-14, None),
    ([5, 6, 4, 5], [3, 4, 2], [2, 3, 3], 1e-2, None),
    ([6, 5, 7], [4, 5], [3, 2], 0.0, [3, 4]),
    ([4, 4, 4, 4, 4], [3, 3, 3, 3], [3, 3, 3, 3], 1e-1, None),
    ([7, 3], [2], [3], 1e-14, None),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_model_matches_oracle_round_tt(case):
    shape, ra, rb, eps, rmax = CASES[case]
    rng = np.random.default_rng(100 + case)
    a, b = _tt(rng, shape, ra), _tt(rng, shape, rb)
    cores, ranks, norm2, disc = hm.hadamard_round(a, b, eps=eps, rmax=rmax)
    oc = orc.round_tt(hm.kronecker(a, b), eps=eps, rmax=rmax)
    assert ranks == [1] + [c.shape[2] for c in oc]
    exact = hm.full(hm.kronecker(a, b))
    mine, ref = hm.full(cores), hm.full(oc)
    nrm = np.linalg.norm(exact)
    e_mine, e_ref = np.linalg.norm(mine - exact) / nrm, np.linalg.norm(ref - exact) / nrm
    assert abs(e_mine - e_ref) <= 1e-8 + 1e-6 * e_ref
    # the energies: ||C||^2 and the sum of the discarded eigenvalues is the rounding's squared error
    assert norm2 == pytest.approx(nrm ** 2, rel=1e-10)
    assert np.sqrt(disc / norm2) == pytest.approx(e_mine, rel=1e-6, abs=1e-7)
    # cores 1..N-1 have orthonormal rows
    for c in cores[1:]:
        M = c.reshape(c.shape[0], -1)
        assert np.allclose(M @ M.T, np.eye(M.shape[0]), atol=1e-10)


def test_gl_recurrence_is_the_left_gram():
    rng = np.random.default_rng(7)
    shape = [3, 4, 5, 3]
    a, b = _tt(rng, shape, [2, 3, 2]), _tt(rng, shape, [3, 2, 2])
    C = hm.kronecker(a, b)
    GL = hm.left_grams(a, b)
    left = np.ones((1, 1))
    for k in range(1, len(shape)):
        left = np.einsum("pr,rix->pix", left, C[k - 1]).reshape(-1, C[k - 1].shape[2])
        assert np.allclose(GL[k], left.T @ left, rtol=1e-12, atol=1e-10)


def test_zero_product_is_rank_one_zeros():
    rng = np.random.default_rng(3)
    shape = [4, 5, 3]
    a, b = _tt(rng, shape, [2, 3]), _tt(rng, shape, [2, 2])
    b[1] = np.zeros_like(b[1])
    cores, ranks, norm2, disc = hm.hadamard_round(a, b)
    assert ranks == [1, 1, 1, 1]
    assert all(not np.any(c) for c in cores)
    assert norm2 == 0.0 and disc == 0.0


def test_model_matches_reference_goldens():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/hadamard_round.npz not generated")
    g = np.load(GOLDEN)
    names = sorted({k.split("/")[0] for k in g.files if k.endswith("/ranks")})
    assert names
    for name in names:
        if f"{name}/a0" not in g.files:
            continue
        N = int(g[f"{name}/N"])
        a = [g[f"{name}/a{k}"] for k in range(N)]
        b = [g[f"{name}/b{k}"] for k in range(N)]
        eps = float(g[f"{name}/eps"])
        rmax = int(g[f"{name}/rmax"])
        cores, ranks, norm2, disc = hm.hadamard_round(a, b, eps=eps, rmax=None if rmax <= 0 else [rmax] * (N - 1))
        assert ranks == list(g[f"{name}/ranks"]), name
        exact = hm.full(hm.kronecker([x.astype(np.float64) for x in a], [x.astype(np.float64) for x in b]))
        nrm = np.linalg.norm(exact)
        err = np.linalg.norm(hm.full(cores) - exact) / nrm if nrm > 0 else 0.0
        assert abs(err - float(g[f"{name}/relerr"])) < 1e-5, name
