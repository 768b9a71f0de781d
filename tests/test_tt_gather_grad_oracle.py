"""CPU: the NumPy restatement of tnb_tt_gather_grad (tests/ttgg_model.py) against an analytic gradient, and its stable
order, chunks and excluded points against their definitions."""
import numpy as np

import ttg_model as tm
import ttgg_model as gm


def _tt(seed, shape, ranks):
    g = np.random.default_rng(seed)
    return [g.standard_normal((ranks[k], shape[k], ranks[k + 1])) for k in range(len(shape))]


def _idx(seed, shape, P, first=0, last=None):
    last = len(shape) if last is None else last
    g = np.random.default_rng(seed)
    return np.stack([g.integers(0, shape[k], P) for k in range(first, last)], axis=1)


def _analytic(cores, idx, gout, first, last):
    """d sum(gout * out) / d G_k by the product rule, one point at a time."""
    grads = [np.zeros_like(cores[k]) for k in range(first, last)]
    for p, row in enumerate(idx):
        sl = [cores[first + m][:, row[m], :] for m in range(last - first)]
        for m in range(last - first):
            left = np.eye(sl[0].shape[0])
            for s in sl[:m]:
                left = left @ s
            right = np.eye(sl[-1].shape[1])
            for s in sl[m + 1:][::-1]:
                right = s @ right
            grads[m][:, row[m], :] += left.T @ gout[:, p, :] @ right.T
    return grads


def test_model_is_the_analytic_gradient():
    for shape, ranks, first, last, P in (([5, 4, 6, 3], [1, 3, 4, 2, 1], 0, 4, 60),
                                         ([5, 4, 6, 3], [2, 3, 4, 2, 3], 1, 3, 40),
                                         ([2] * 6, [1, 2, 3, 2, 3, 2, 1], 0, 6, 2000),
                                         ([7], [1, 1], 0, 1, 30)):
        cores = _tt(1, shape, ranks)
        idx = _idx(2, shape, P, first, last)
        gout = np.random.default_rng(3).standard_normal((ranks[first], P, ranks[last]))
        got = gm.grad(cores, idx, gout, first, last)
        want = _analytic(cores, idx, gout, first, last)
        for g, w in zip(got, want):
            np.testing.assert_allclose(g, w, rtol=1e-11, atol=1e-11)


def test_excluded_points_add_nothing():
    shape, ranks = [5, 4, 6], [1, 3, 4, 1]
    cores = _tt(4, shape, ranks)
    idx = _idx(5, shape, 50)
    gout = np.random.default_rng(6).standard_normal((1, 51, 1))
    bad = np.vstack([idx[:20], [[0, 4, 1]], idx[20:]])
    keep = np.delete(gout, 20, axis=1)
    for g, w in zip(gm.grad(cores, bad, gout), gm.grad(cores, idx, keep)):
        np.testing.assert_allclose(g, w, rtol=1e-13, atol=1e-13)
    assert (gm.buckets(bad, shape, 0, 3)[:, 20] == np.array(shape)).all()


def test_stable_order_and_chunks():
    b = np.array([3, 1, 3, 0, 1, 3, 4, 4, 3])
    np.testing.assert_array_equal(gm.order(b), [3, 1, 4, 0, 2, 5, 8, 6, 7])
    ch = gm.chunks(b, 4, 2, 4)
    assert ch == [(0, 0, 2), (1, 2, 4), (3, 6, 4), (3, 10, 4), (4, 14, 4)]
    assert len(ch) <= gm.chunk_bound(18, 4, 4)
    rows = 2 * 4
    assert sum(-(-c // 4) for c in (8,)) <= gm.slot_bound(rows, 4) + 2


def test_paths_and_kernels():
    r = [1, 16, 24, 300, 20, 1]
    assert gm.mode_paths(r, 0, 5) == [tm.RANK_MIN, tm.TC, tm.RANK_MAX, tm.RANK_MAX, tm.RANK_MIN]
    assert gm.kernels([1, 16, 24, 20, 1], 1, 3) == {"ttgg_reduce_tc_kernel", "ttg_step_tc_kernel"}
    assert gm.kernels([1, 1], 0, 1) == {"ttgg_reduce_generic_kernel"}
    assert gm.launches([7], [[1, 1]], 0, 1) == 1 + 4 + (0 + 1 + 0 + 1 + 2 + 0)
