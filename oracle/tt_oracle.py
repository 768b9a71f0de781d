"""CPU oracle for the tntorch decomposition / rounding hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``tntorch_b200/`` may import this file;
only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` legs do.  It is a plain NumPy (LAPACK) restatement of the
reference's algorithm, function by function, each citing the reference file:line
it follows.  Parity is PINNED: ``oracle/gen_golden.py`` imports the real reference
from ``/root/reference`` (in the build container) and stores its outputs under
``tests/golden/``; ``tests/test_oracle.py`` checks this file against them.

The reference computes with ``torch.linalg.{qr,svd,eigh}`` (LAPACK on CPU); NumPy
calls the same LAPACK drivers (geqrf/orgqr, gesdd, syevd), so the restatement
agrees with the reference to rounding.
"""
from __future__ import annotations

import numpy as np

__all__ = [
    "full_rank_tt",
    "left_orthogonalize",
    "orthogonalize_to_last",
    "truncated_svd",
    "round_tt",
    "tt_svd",
    "tt_reconstruct",
    "relative_error",
    "py_maxvol",
    "py_rect_maxvol",
    "cp_to_tt",
    "factor_orthogonalize",
    "orthogonalize",
    "round_tt_tucker",
    "round_tucker",
    "round",
    "tucker_from_dense",
    "tucker_eps",
    "tucker_core",
    "tucker_full",
]


# --------------------------------------------------------------------------- #
# dense -> exact full-rank TT          (reference: tntorch/tensor.py:10-104)
# --------------------------------------------------------------------------- #
def full_rank_tt(data: np.ndarray):
    """Exact TT of a dense array with identity flanks (tensor.py:10-104, non-batch
    branch: 36-64 identity-left case, 86-96 data-core case, 101-103 last core)."""
    shape = data.shape
    N = data.ndim
    dtype = data.dtype
    result = []
    resh = data.reshape(shape[0], -1)
    for n in range(1, N):
        if resh.shape[0] < resh.shape[1]:
            eye = np.eye(resh.shape[0], dtype=dtype)
            result.append(eye.reshape(resh.shape[0] // shape[n - 1], shape[n - 1], resh.shape[0]))
            resh = resh.reshape(resh.shape[0] * shape[n], resh.shape[1] // shape[n])
        else:
            result.append(resh.reshape(resh.shape[0] // shape[n - 1], shape[n - 1], resh.shape[1]))
            eye = np.eye(resh.shape[1], dtype=dtype)
            resh = eye.reshape(resh.shape[1] * shape[n], resh.shape[1] // shape[n])
    result.append(resh.reshape(resh.shape[0] // shape[N - 1], shape[N - 1], 1))
    return result


# --------------------------------------------------------------------------- #
# QR orthogonalisation sweeps          (reference: tntorch/tensor.py:1800-1909)
# --------------------------------------------------------------------------- #
def left_orthogonalize(cores, mu: int):
    """tensor.py:1800-1833: thin QR of the left unfolding, R pushed right."""
    assert 0 <= mu < len(cores) - 1
    c = cores[mu]
    Q, R = np.linalg.qr(c.reshape(-1, c.shape[-1]))  # tensor.py:1816
    cores[mu] = Q.reshape(c.shape[:-1] + (Q.shape[1],))
    nxt = cores[mu + 1]
    cores[mu + 1] = (R @ nxt.reshape(nxt.shape[0], -1)).reshape((R.shape[0],) + nxt.shape[1:])
    return R


def right_orthogonalize(cores, mu: int):
    """tensor.py:1835-1879: QR of the transposed right unfolding, L pushed left."""
    assert 1 <= mu < len(cores)
    c = cores[mu]
    Q, L = np.linalg.qr(c.reshape(c.shape[0], -1).T)
    L = L.T
    Q = Q.T
    cores[mu] = Q.reshape((Q.shape[0],) + c.shape[1:])
    prv = cores[mu - 1]
    cores[mu - 1] = (prv.reshape(-1, prv.shape[-1]) @ L).reshape(prv.shape[:-1] + (L.shape[1],))
    return L


def orthogonalize_to_last(cores):
    """tensor.py:1881-1909 with mu = N-1 (what round_tt calls at tensor.py:2033)."""
    for i in range(len(cores) - 1):
        left_orthogonalize(cores, i)


# --------------------------------------------------------------------------- #
# two-factor rank-revealing split      (reference: tntorch/round.py:52-187)
# --------------------------------------------------------------------------- #
def truncated_svd(M, delta=None, eps=None, rmax=None, left_ortho=True, algorithm="svd"):
    """round.py:52-187, non-batch path.  Returns (left [m,r], right [r,n])."""
    if delta is not None and eps is not None:
        raise ValueError("Provide either `delta` or `eps`")  # round.py:77-78
    if delta is None and eps is not None:
        delta = eps * float(np.linalg.norm(M))
    if delta is None and eps is None:
        delta = 0
    if rmax is None:
        rmax = np.iinfo(np.int32).max
    assert rmax >= 1
    assert algorithm in ("svd", "eig")

    if algorithm == "svd":
        U, S, _ = np.linalg.svd(M, full_matrices=False)  # round.py:96 (only U,S are used)
        vecs, sing = U, S
        which = "left"
    else:  # round.py:101-135
        if M.shape[0] <= M.shape[1]:
            gram = M @ M.T
            which = "left"
        else:
            gram = M.T @ M
            which = "right"
        w, v = np.linalg.eigh(gram)
        w = np.where(w < 0, np.zeros_like(w) + 1e-8, w)  # round.py:118
        w = np.sqrt(w)
        idx = np.argsort(w)[::-1]
        vecs, sing = v[:, idx], w[idx]

    if sing[0] < 1e-13:  # round.py:137-145 zero-matrix special case
        return np.zeros((M.shape[0], 1), M.dtype), np.zeros((1, M.shape[1]), M.dtype)

    S2 = sing**2
    where = np.where(np.cumsum(S2[::-1]) <= delta**2)[0]  # round.py:151-152
    if len(where) == 0:
        rank = max(1, int(min(rmax, len(S2))))
    else:
        rank = max(1, int(min(rmax, len(S2) - 1 - where[-1])))
    left = vecs[:, :rank]
    s = sing[:rank]
    if which == "left":
        if left_ortho:
            M2 = left.T @ M
        else:
            M2 = (1.0 / s)[:, None] * left.T @ M  # round.py:166-172
            left = left * s
    else:
        if left_ortho:
            M2 = M @ (left * (1.0 / s)[None, :])
            left, M2 = M2, (left @ np.diag(s)).T
        else:
            M2 = M @ left
            left, M2 = M2, left.T
    return left.astype(M.dtype, copy=False), M2.astype(M.dtype, copy=False)


# --------------------------------------------------------------------------- #
# TT rounding                          (reference: tntorch/tensor.py:2008-2083)
# --------------------------------------------------------------------------- #
def round_tt(cores, eps=1e-14, rmax=None, algorithm="svd"):
    """In-place TT rounding: QR sweep L->R, then SVD truncation R->L."""
    N = len(cores)
    if not hasattr(rmax, "__len__"):
        rmax = [rmax] * (N - 1)
    assert len(rmax) == N - 1
    orthogonalize_to_last(cores)  # tensor.py:2033
    delta = eps / max(1.0, np.sqrt(N - 1)) * float(np.linalg.norm(cores[-1]))  # tensor.py:2039-2051
    for mu in range(N - 1, 0, -1):  # tensor.py:2053
        c = cores[mu]
        M = c.reshape(c.shape[0], -1)
        left, right = truncated_svd(M, delta=delta, rmax=rmax[mu - 1], left_ortho=False, algorithm=algorithm)
        cores[mu] = right.reshape(-1, c.shape[1], c.shape[2])
        cores[mu - 1] = np.einsum("ijk,kl->ijl", cores[mu - 1], left)  # tensor.py:2081-2083
    return cores


def tt_svd(data: np.ndarray, ranks_tt=None, eps=None, algorithm="svd"):
    """``tn.Tensor(data, ranks_tt=r)`` (tensor.py:401-408): full-rank TT + round_tt.
    With ``eps`` it follows the ``eps`` branch (tensor.py:436-439 -> round -> round_tt)."""
    cores = full_rank_tt(np.asarray(data))
    if eps is not None:
        return round_tt(cores, eps=eps, rmax=None, algorithm=algorithm)
    return round_tt(cores, rmax=ranks_tt, algorithm=algorithm)


# --------------------------------------------------------------------------- #
# reconstruction + error               (tensor.py:1639-1687, metrics.py:135-151)
# --------------------------------------------------------------------------- #
def tt_reconstruct(cores, dtype=np.float64):
    f = np.ones((1, cores[0].shape[0]), dtype=dtype)
    shape = []
    for c in cores:
        shape.append(c.shape[1])
        f = (f @ c.reshape(c.shape[0], -1).astype(dtype)).reshape(-1, c.shape[2])
    return f.sum(axis=-1).reshape(shape) if f.shape[-1] > 1 else f[..., 0].reshape(shape)


def relative_error(gt: np.ndarray, cores) -> float:
    """‖gt − T̂‖_F/‖gt‖_F with T̂ reconstructed and differenced in fp64."""
    gt64 = np.asarray(gt, dtype=np.float64)
    return float(np.linalg.norm(gt64 - tt_reconstruct(cores)) / np.linalg.norm(gt64))


# --------------------------------------------------------------------------- #
# Tucker factors, CP cores, Tucker rounding   (reference: tntorch/tensor.py:1717-2098)
# A tensor is (cores, Us): cores [r0, S, r1] (TT) or [S, R] (CP), Us[n] [I, S] or None.
# --------------------------------------------------------------------------- #
def _cp_factor_to_core(factor):
    """tensor.py:1741-1765, non-batch: a CP factor [I, R] -> the TT core [R, I, R] whose slices are diag(factor[i])."""
    if factor.ndim == 3:  # already a TT core (:1741-1742)
        return factor
    I, R = factor.shape
    core = np.zeros((R, I, R), dtype=factor.dtype)
    core[np.arange(R), :, np.arange(R)] = factor.T
    return core


def cp_to_tt(cores):
    """tensor.py:1728-1740 (factor=None): the first CP factor becomes [1, I, R], the middle ones diagonal [R, I, R]
    cores, the last [R, I, 1].  In place on the list; returns it."""
    if cores[0].ndim == 2:
        cores[0] = cores[0][None, ...]
    for mu in range(1, len(cores) - 1):
        cores[mu] = _cp_factor_to_core(cores[mu])
    if cores[-1].ndim == 2:
        cores[-1] = cores[-1].T[..., None]
    return cores


def factor_orthogonalize(cores, Us, mu: int):
    """tensor.py:1771-1798: U_mu = Q R, the core (TT or CP) absorbs R along its mode index."""
    if Us[mu] is None:
        return
    Q, R = np.linalg.qr(Us[mu])  # :1783
    Us[mu] = Q
    if cores[mu].ndim == 2:
        cores[mu] = np.einsum("jk,aj->ak", cores[mu], R)  # :1796
    else:
        cores[mu] = np.einsum("ijk,aj->iak", cores[mu], R)  # :1798


def orthogonalize(cores, Us, mu: int):
    """tensor.py:1881-1909 with the factor pushes of left_/right_orthogonalize (:1815, :1850): CP cores become TT
    cores, then left QRs for 0..mu-1 and right QRs for N-1..mu+1.  Returns (R, L) as the reference does."""
    N = len(cores)
    if mu < 0:
        mu += N
    cp_to_tt(cores)
    R = np.ones((1, 1))
    L = np.ones((1, 1))
    for i in range(mu):
        factor_orthogonalize(cores, Us, i)
        R = left_orthogonalize(cores, i)
    for i in range(N - 1, mu, -1):
        factor_orthogonalize(cores, Us, i)
        L = right_orthogonalize(cores, i)
    return R, L


def round_tt_tucker(cores, Us, eps=1e-14, rmax=None, algorithm="svd"):
    """tensor.py:2008-2083 on a tensor with Tucker factors: CP cores become TT cores (:2031), orthogonalize(N-1)
    pushes the factors of modes 0..N-2 into their cores (:2033; the last factor stays as it is), then the TT
    truncation sweep.  In place on the lists; returns them."""
    N = len(cores)
    cp_to_tt(cores)
    for mu in range(N - 1):
        factor_orthogonalize(cores, Us, mu)
    round_tt(cores, eps=eps, rmax=rmax, algorithm=algorithm)
    return cores, Us


def round_tucker(cores, Us, eps=1e-14, rmax=None, dim="all", algorithm="svd"):
    """tensor.py:1911-2006, non-batch.  In place on the lists `cores` and `Us`.  Returns, per mode in the order the
    reference visits them (N-1 down to 0), what its factor split saw: the QR shape (r0 r1 x S), k, I, whether the mode
    had a factor and a CP core before the call, the budget and rmax of its truncated_svd, the singular values of the
    I x k matrix it split, and the rank it kept."""
    N = len(cores)
    if not hasattr(rmax, "__len__"):
        rmax = [rmax] * N
    assert len(rmax) == N
    if dim == "all":
        dim = range(N)
    if not hasattr(dim, "__len__"):
        dim = [dim] * N
    had_U = [U is not None for U in Us]
    was_cp = [c.ndim == 2 for c in cores]
    for m in dim:  # :1942-1943: the CP factors of `dim` become diagonal cores, boundary ones included
        cores[m] = _cp_factor_to_core(cores[m])
    orthogonalize(cores, Us, -1)  # :1944
    budget = eps / np.sqrt(len(dim))  # :1990
    info = []
    for mu in range(N - 1, -1, -1):
        c = cores[mu]
        r0, S, r1 = c.shape
        if Us[mu] is None:
            Us[mu] = np.eye(S, dtype=c.dtype)  # :1946-1957
        Q, R = np.linalg.qr(c.transpose(0, 2, 1).reshape(-1, S))  # :1976-1983
        cores[mu] = Q.reshape(r0, r1, -1).transpose(0, 2, 1)
        Us[mu] = Us[mu] @ R.T  # :1985
        sv = np.linalg.svd(Us[mu], compute_uv=False)
        left, right = truncated_svd(Us[mu], eps=budget, rmax=rmax[mu], left_ortho=True, algorithm=algorithm)  # :1988
        Us[mu] = left
        cores[mu] = np.einsum("ijk,aj->iak", cores[mu], right)  # :2002
        info.append(dict(mu=mu, rows=r0 * r1, S=S, k=Q.shape[1], I=Us[mu].shape[0], had_U=had_U[mu], cp=was_cp[mu],
                         eps=budget, rmax=rmax[mu], sv=sv, rank=left.shape[1]))
        if mu > 0:
            factor_orthogonalize(cores, Us, mu)  # :2006 right_orthogonalize(mu)
            right_orthogonalize(cores, mu)
    return info


def tucker_core(cores):
    """tensor.py:1565-1574: the dense core tensor of the TT (or CP) cores, factors left out."""
    return tt_reconstruct(cp_to_tt(list(cores)))


def tucker_full(cores, Us):
    """The dense tensor of (cores, Us): each factor absorbed into its core (tensor.py:1576-1627, 'ijk,aj->iak'), the
    chain contracted with the boundary ranks summed (tensor.py:1639-1687)."""
    cs = []
    for c, U in zip(cp_to_tt(list(cores)), Us):
        c = np.asarray(c, dtype=np.float64)
        cs.append(c if U is None else np.einsum("ijk,aj->iak", c, np.asarray(U, dtype=np.float64)))
    f = np.ones((1, cs[0].shape[0]))
    for c in cs:
        f = (f @ c.reshape(c.shape[0], -1)).reshape(-1, c.shape[2])
    return f.sum(axis=-1).reshape([c.shape[1] for c in cs])


def round(cores, Us, eps=1e-14, rmax=None, algorithm="svd"):
    """tensor.py:2085-2098: TT rounding, then Tucker rounding with the budget left over, (1 + eps) / (1 + reached) - 1,
    when the TT rounding reached less than eps.  In place on the lists; returns (reached, round_tucker's info or
    None)."""
    before = tucker_full(cores, Us)
    round_tt_tucker(cores, Us, eps, rmax=rmax, algorithm=algorithm)
    after = tucker_full(cores, Us)
    reached = float(np.linalg.norm(before - after) / np.linalg.norm(before))  # metrics.relative_error (:2096)
    info = None
    if reached < eps:
        info = round_tucker(cores, Us, (1 + eps) / (1 + reached) - 1, rmax=rmax, algorithm=algorithm)
    return reached, info


def tucker_from_dense(data, ranks_tucker, ranks_tt=None, algorithm="svd"):
    """tn.Tensor(data, ranks_tucker=, ranks_tt=) (tensor.py:401-408): the exact TT (_full_rank_tt), round_tucker with
    rmax = ranks_tucker, then round_tt with rmax = ranks_tt.  Returns (cores, Us, round_tucker's info)."""
    cores = full_rank_tt(np.asarray(data))
    Us = [None] * len(cores)
    info = round_tucker(cores, Us, rmax=ranks_tucker, algorithm=algorithm)
    if ranks_tt is not None:
        round_tt_tucker(cores, Us, rmax=ranks_tt, algorithm=algorithm)
    return cores, Us, info


def tucker_eps(data, eps, algorithm="svd"):
    """tn.Tensor(data, eps=) (tensor.py:436-439 -> round, :2085-2098): _full_rank_tt + round_tt(eps), which is
    tt_svd(eps), then round_tucker with the budget left over.  Returns (cores, Us, reached, round_tucker's info or
    None)."""
    cores = tt_svd(np.asarray(data), eps=eps, algorithm=algorithm)
    Us = [None] * len(cores)
    reached = relative_error(data, cores) if len(cores) >= 2 else 0.0
    info = None
    if reached < eps:
        info = round_tucker(cores, Us, (1 + eps) / (1 + reached) - 1, algorithm=algorithm)
    return cores, Us, reached, info


# --------------------------------------------------------------------------- #
# maxvol                               (reference: tntorch/maxvol.py:114-170)
# --------------------------------------------------------------------------- #
def py_maxvol(A, tol=1.05, max_iters=100):
    """Dominant r×r submatrix of an N×r matrix: LU-pivot initialisation followed by
    greedy row swaps with rank-1 updates of the coefficient matrix
    (maxvol.py:114-170; LAPACK getrf/trtrs + BLAS ger there, scipy here).  The
    coefficient matrix is kept transposed (r×N) like the reference so that the
    flat ``argmax`` breaks ties the same way."""
    from scipy.linalg import lu_factor, solve_triangular

    A = np.asarray(A, dtype=np.float64)
    if tol < 1:
        tol = 1.0
    N, r = A.shape
    if N <= r:
        return np.arange(N, dtype=np.int32), np.eye(N, dtype=A.dtype)
    lu, piv = lu_factor(A)  # getrf of the N×r matrix (maxvol.py:135)
    index = np.arange(N, dtype=np.int32)
    for i in range(r):  # maxvol.py:137-141
        tmp = index[i]
        index[i] = index[piv[i]]
        index[piv[i]] = tmp
    H = lu[:r]
    # solve A = C H with H in LU form: two triangular solves (maxvol.py:145-148)
    C = solve_triangular(H, A.T.copy(), trans=1, lower=False)
    C = solve_triangular(H, C, trans=1, lower=True, unit_diagonal=True)  # r×N
    i, j = divmod(int(np.abs(C).argmax()), N)
    iters = 0
    while abs(C[i, j]) > tol and iters < max_iters:  # maxvol.py:160-169
        index[i] = j
        tmp_row = C[i].copy()
        tmp_column = C[:, j].copy()
        tmp_column[i] -= 1.0
        alpha = -1.0 / C[i, j]
        C += alpha * np.outer(tmp_column, tmp_row)
        iters += 1
        i, j = divmod(int(np.abs(C).argmax()), N)
    return index[:r].copy(), C.T


def py_rect_maxvol(A, tol=1.0, maxK=None, min_add_K=None, minK=None, start_maxvol_iters=10):
    """Rectangular 2-volume maximisation (maxvol.py:30-111, identity_submatrix=True, top_k_index = N): maxvol with
    `start_maxvol_iters` swaps (:73), then rows are added while the largest squared row norm of the coefficient
    matrix exceeds tol^2 (K < maxK) or K < minK, each by the rank-1 Sherman-Woodbury-Morrison update of :94-103."""
    A = np.asarray(A, dtype=np.float64)
    tol2 = tol ** 2
    N, r = A.shape
    if N <= r:
        return np.arange(N, dtype=np.int32), np.eye(N, dtype=A.dtype)
    if maxK is None or maxK > N:  # parameter normalisation, maxvol.py:54-66
        maxK = N
    if maxK < r:
        maxK = r
    if minK is None or minK < r:
        minK = r
    if minK > N:
        minK = N
    if min_add_K is not None:
        minK = max(minK, r + min_add_K)
    if minK > maxK:
        minK = maxK
    index = np.zeros(N, dtype=np.int32)
    chosen = np.ones(N)
    tmp_index, C = py_maxvol(A, 1.05, start_maxvol_iters)
    index[:r] = tmp_index
    chosen[tmp_index] = 0
    C = C.copy()
    row_norm_sqr = chosen * np.sum(C * C, axis=1)
    i = int(np.argmax(row_norm_sqr))
    K = r
    while (row_norm_sqr[i] > tol2 and K < maxK) or K < minK:
        index[K] = i
        chosen[i] = 0
        c = C[i].copy()
        v = C @ c
        l = 1.0 / (1 + v[i])
        C = np.hstack([C - l * np.outer(v, c), (l * v)[:, None]])
        row_norm_sqr = (row_norm_sqr - l * v * v) * chosen
        i = int(np.argmax(row_norm_sqr))
        K += 1
    C[index[:K]] = np.eye(K)
    return index[:K].copy(), C
