"""CPU: the NumPy restatement oracle.matrix_oracle.tt_multiply equals the reference's tt_multiply (matrix.py:420-443) on
every golden case, and X @ M with M formed from the same cores."""
import os

import numpy as np
import pytest

from oracle import matrix_oracle as orc

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(REPO, "tests", "golden", "tt_multiply.npz"))
NAMES = sorted({k.split("/")[0] for k in G.files})


def golden(name):
    cores = [G[f"{name}/core{k}"] for k in range(int(G[f"{name}/d"]))]
    return cores, G[f"{name}/X"], G[f"{name}/Y"]


def dense_matrix(cores):
    """M (I x O) from cores [r, i, o, r'], rows (i_0 .. i_{d-1}) and columns (o_0 .. o_{d-1}) row-major."""
    M = np.ones((1, 1, 1))
    for c in cores:
        M = np.einsum("abr,rios->aibos", M, c).reshape(M.shape[0] * c.shape[1], M.shape[1] * c.shape[2], c.shape[3])
    return M[:, :, 0]


def test_the_golden_cases_cover_the_issue():
    assert {"ref_f64", "d1_f64", "d4_unit_modes_f64", "x3d_f64", "f32_d2", "f32_d3"} <= set(NAMES)
    assert G["x3d_f64/X"].ndim == 3
    assert G["ref_f64/X"].shape == (30, 33) and G["ref_f64/Y"].shape == (30, 46)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_equals_reference(name):
    cores, X, Y = golden(name)
    got = orc.tt_multiply(cores, X)
    assert got.shape == Y.shape and got.dtype == Y.dtype
    tol = 1e-12 if Y.dtype == np.float64 else 1e-6
    assert np.linalg.norm(got - Y) <= tol * np.linalg.norm(Y), name


@pytest.mark.parametrize("name", NAMES)
def test_oracle_is_x_times_m(name):
    cores, X, _ = golden(name)
    c64 = [c.astype(np.float64) for c in cores]
    want = X.astype(np.float64).reshape(-1, dense_matrix(c64).shape[0]) @ dense_matrix(c64)
    got = orc.tt_multiply(c64, X.astype(np.float64))
    assert np.linalg.norm(got - want) <= 1e-12 * np.linalg.norm(want)


def test_oracle_refuses_a_vector():
    cores, X, _ = golden("d1_f64")
    with pytest.raises(AssertionError):
        orc.tt_multiply(cores, X[0])
