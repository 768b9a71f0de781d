"""CPU oracle for the TT-matrix product (reference: tntorch/matrix.py:420-443).

TEST INFRASTRUCTURE ONLY, like ``oracle/tt_oracle.py``: nothing under ``tntorch_b200/`` imports it.  A plain NumPy
restatement of the reference's ``tt_multiply``; ``tests/test_tt_multiply_oracle.py`` pins it to the reference's outputs
stored by ``oracle/gen_matrix.py`` in ``tests/golden/tt_multiply.npz``.
"""
from __future__ import annotations

import numpy as np

__all__ = ["tt_multiply"]


def tt_multiply(cores, X: np.ndarray) -> np.ndarray:
    """X viewed as [b, I] times the TT-matrix of cores [r_k, i_k, o_k, r_{k+1}] (matrix.py:420-443): X.T, then one
    contraction per core of the leading input mode and the trailing rank, appending (o_k, r_{k+1})."""
    assert X.ndim > 1
    idims = [c.shape[1] for c in cores]
    b = X.reshape(-1, int(np.prod(idims))).shape[0]
    res = X.reshape(b, -1).T.reshape(idims[0], -1)
    res = np.einsum("id,lior->ldor", res, cores[0])
    for k in range(1, len(cores)):
        res = res.reshape(idims[k], -1, cores[k].shape[0])
        res = np.einsum("idr,riob->dob", res, cores[k])
    return res.reshape(b, -1)
