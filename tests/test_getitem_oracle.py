"""CPU: the goldens of Tensor.__getitem__ (tests/golden/getitem.npz, the reference's own results from
oracle/gen_getitem.py) against NumPy: every value a key gives is the dense tensor indexed by NumPy with the same key
(index arrays are contiguous, so NumPy places their axis where the reference does), and the values at a P x N matrix
are the fp64 chain of tests/ttg_model.py, the computation tnb_tt_gather runs."""
import os

import numpy as np
import pytest
import torch

import ttg_model as tm
from oracle import getitem_cases as gc

GOLD = os.path.join(os.path.dirname(__file__), "golden", "getitem.npz")


def case_tensor(g, spec, dname):
    """(cores, Us, batch) as NumPy arrays."""
    t = gc.tensor(spec, gc.DTYPES[dname])
    if t is None:
        n = int(g[f"{spec}/{dname}/n"])
        return [g[f"{spec}/{dname}/core{k}"] for k in range(n)], [g[f"{spec}/{dname}/U{k}"] for k in range(n)], False
    cores, Us, batch = t
    return [c.numpy() for c in cores], Us, batch


def dense(cores, Us, batch):
    """The full tensor in fp64."""
    if batch:
        return np.stack([dense([c[b] for c in cores], Us, False) for b in range(cores[0].shape[0])])
    if cores[0].ndim == 2:  # CP factors [I, R]: sum_r prod_k A_k[i_k, r]
        f = np.asarray(cores[0], np.float64)
        for c in cores[1:]:
            f = np.einsum("...r,ir->...ir", f, np.asarray(c, np.float64))
        return f.sum(-1)
    cs = []
    for k, c in enumerate(cores):
        c = np.asarray(c, np.float64)
        if Us is not None and Us[k] is not None:
            c = np.einsum("ijk,aj->iak", c, np.asarray(Us[k], np.float64))
        cs.append(c)
    f = cs[0]
    for c in cs[1:]:
        f = np.tensordot(f, c, axes=([-1], [0]))
    return f.sum(axis=(0, -1)) if f.shape[0] * f.shape[-1] > 1 else f[0, ..., 0]


def numpy_key(key):
    if isinstance(key, np.ndarray) and key.ndim == 2:
        return tuple(key[:, j] for j in range(key.shape[1]))
    if isinstance(key, torch.Tensor):
        return numpy_key(key.numpy())
    if isinstance(key, tuple):
        return tuple(k.numpy() if isinstance(k, torch.Tensor) else (np.asarray(k) if isinstance(k, list) else k)
                     for k in key)
    if isinstance(key, list):
        return (np.asarray(key),)
    return key


CASES = [(n, d) for n in gc.KEYS for d in gc.DTYPES]


@pytest.mark.parametrize("name,dname", CASES)
def test_golden_is_numpy_indexing(name, dname):
    g = np.load(GOLD)
    spec, key = gc.KEYS[name]
    kind = str(g[f"{name}/{dname}/kind"])
    if kind not in ("tensor", "scalar"):
        assert kind in ("IndexError", "ValueError")
        return
    full = dense(*case_tensor(g, spec, dname))
    want = full[numpy_key(key("cpu"))]
    tol = 1e-12 if dname == "f64" else 1e-5
    got = g[f"{name}/{dname}/value"]
    assert got.shape == np.shape(want), (got.shape, np.shape(want))
    assert np.abs(got - want).max() <= tol * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("dname", list(gc.DTYPES))
def test_matrix_values_are_the_model_chain(dname):
    g = np.load(GOLD)
    for name in ("matrix_numpy", "rank1_matrix"):
        spec, key = gc.KEYS[name]
        cores, _, _ = case_tensor(g, spec, dname)
        got = tm.gather(cores, key("cpu"))
        assert got.shape == (1, key("cpu").shape[0], 1)
        tol = 1e-12 if dname == "f64" else 1e-5
        want = g[f"{name}/{dname}/value"]
        assert np.abs(got[0, :, 0] - want).max() <= tol * max(1.0, np.abs(want).max())


def test_inner_block_is_the_model_range():
    """t[:, i, j, :] of the reference is the [r1, P, r3] range product of modes 1 and 2."""
    g = np.load(GOLD)
    spec, key = gc.KEYS["inner_block"]
    cores, _, _ = case_tensor(g, spec, "f64")
    k = key("cpu")
    idx = np.stack([k[1], k[2]], axis=1)
    block = tm.gather(cores, idx, 1, 3)
    np.testing.assert_array_equal(g["inner_block/f64/core_shapes"][1][:3], block.shape)
