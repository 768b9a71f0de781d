"""fp64 NumPy statement of TT-cross (tntorch cross.py:138-529), one sweep step at a time, with the decision margin of every
maxvol choice.  Shares no code with `tntorch_b200/cross.py`, `cross_batch.py` or the kernels: samples come from indexing
the grid (or evaluating the input TTs) at the multi-indices of the index sets, the QR is `np.linalg.qr`, the row choice is
`oracle.tt_oracle.py_maxvol` / `py_rect_maxvol`, and the interpolation core is `np.linalg.solve`.

Index sets use the reference's layout: lsets[j] is [R_j, j + 1] with a leading 0 column, rsets[j] is [R_{j+1}, N - j]
with a trailing 0 column.

A margin is the relative distance of a decision from flipping:
  - LU pivot search (maxvol.py:135):   (best - second) / best over the |values| of the pivot column
  - swap phase (maxvol.py:150-169):    the same over |C|, and |best - tol| / tol for the stop test
  - rect_maxvol extension (:68-103):   the same over the squared row norms, and |best - tol^2| / tol^2
Two correct implementations that differ by rounding make the same choices wherever every margin is well above the
rounding level, so index sets are compared exactly only where `margin` exceeds a stated level.  A step also records
`cond` = sigma_min / sigma_max of its sample matrix: duplicate fibres (random initial right sets can repeat a row) make
it exactly rank deficient, and then Q's completion, and every choice made from it, is rounding noise.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle.tt_oracle import py_maxvol, py_rect_maxvol


def _gap(vals):
    """(best - second) / best over non-negative values (inf for fewer than two candidates)."""
    vals = np.asarray(vals, dtype=np.float64).ravel()
    if vals.size < 2:
        return np.inf
    second, best = np.partition(vals, -2)[-2:]
    return 0.0 if best == 0 else float((best - second) / best)


def _lu_pivots(A):
    """Unblocked partial-pivoting LU of the N x r matrix: pivot rows in getrf order and each pivot search's margin."""
    B = np.array(A, dtype=np.float64)
    N, r = B.shape
    perm = np.arange(N)
    margins = []
    for k in range(r):
        col = np.abs(B[k:, k])
        margins.append(_gap(col))
        p = k + int(np.argmax(col))
        if p != k:
            B[[k, p]] = B[[p, k]]
            perm[[k, p]] = perm[[p, k]]
        if B[k, k] != 0:
            B[k + 1:, k] /= B[k, k]
        B[k + 1:, k + 1:] -= np.outer(B[k + 1:, k], B[k, k + 1:])
    return perm[:r].copy(), margins


def _swaps(A, index, tol, max_iters):
    """The greedy swap phase from the pivot rows `index`: final index, swap count, and per-decision margins."""
    N, r = A.shape
    index = np.array(index)
    C = np.linalg.solve(A[index].T, A.T)  # r x N, the reference's transposed layout
    argm, stop = [], []
    iters = 0
    while True:
        a = np.abs(C)
        flat = int(a.argmax())
        i, j = divmod(flat, N)
        best = a[i, j]
        if iters >= max_iters:
            break
        stop.append(abs(best - tol) / tol)
        if not best > tol:
            break
        argm.append(_gap(a))
        index[i] = j
        row = C[i].copy()
        col = C[:, j].copy()
        col[i] -= 1.0
        C += (-1.0 / C[i, j]) * np.outer(col, row)
        iters += 1
    return index, iters, argm, stop


def maxvol(A, tol=1.05, max_iters=100):
    """py_maxvol(A, tol, max_iters) plus its swap count and margins.
    Returns (index int32 [r], C [N, r], info) with info = {iters, lu, swap, stop, margin}; `margin` is the smallest."""
    A = np.asarray(A, dtype=np.float64)
    index, C = py_maxvol(A, tol, max_iters)
    N, r = A.shape
    info = dict(iters=0, lu=[], swap=[], stop=[], margin=np.inf)
    if N <= r:
        return index, C, info
    t = max(float(tol), 1.0)
    piv, lu = _lu_pivots(A)
    idx2, iters, swap, stop = _swaps(A, piv, t, max_iters)
    info.update(iters=iters, lu=lu, swap=swap, stop=stop, margin=min(lu + swap + stop + [np.inf]))
    if info["margin"] > 1e-9:  # away from ties the restatement must agree with py_maxvol
        assert np.array_equal(idx2, index), (idx2, index)
    return index, C, info


def rect_params(N, r, maxK=None, min_add_K=None, minK=None):
    """maxvol.py:54-66: (minK, maxK) after normalisation."""
    if maxK is None or maxK > N:
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
    return minK, maxK


def rect_maxvol(A, tol=1.0, maxK=None, min_add_K=None, minK=None, start_maxvol_iters=10):
    """py_rect_maxvol plus margins: those of the start maxvol (tol 1.05) and of every row-adding decision."""
    A = np.asarray(A, dtype=np.float64)
    index, C = py_rect_maxvol(A, tol, maxK, min_add_K, minK, start_maxvol_iters)
    N, r = A.shape
    info = dict(margin=np.inf, add=[], stop=[], start=None)
    if N <= r:
        return index, C, info
    lo, hi = rect_params(N, r, maxK, min_add_K, minK)
    i0, C0, start = maxvol(A, 1.05, start_maxvol_iters)
    tol2 = tol ** 2
    chosen = np.ones(N)
    chosen[i0] = 0
    Cw = C0.copy()
    norms = chosen * np.sum(Cw * Cw, axis=1)
    K = r
    add, stop = [], []
    idx2 = list(i0)
    while True:
        i = int(np.argmax(norms))
        if K >= lo and K < hi:  # the tolerance decides
            stop.append(abs(norms[i] - tol2) / tol2 if tol2 > 0 else np.inf)
        if not ((norms[i] > tol2 and K < hi) or K < lo):
            break
        add.append(_gap(norms[chosen > 0]))
        idx2.append(i)
        chosen[i] = 0
        c = Cw[i].copy()
        v = Cw @ c
        l = 1.0 / (1 + v[i])
        Cw = np.hstack([Cw - l * np.outer(v, c), (l * v)[:, None]])
        norms = (norms - l * v * v) * chosen
        K += 1
    info.update(start=start, add=add, stop=stop, margin=min([start["margin"]] + add + stop))
    if info["margin"] > 1e-9:  # away from ties the restatement must agree with py_rect_maxvol
        assert np.array_equal(idx2, index), (idx2, index)
    return index, C, info


# --------------------------------------------------------------------------- sampling
def tt_values(cores, M):
    """Values of the TT `cores` (numpy [r, I, r']) at the multi-indices M [P, N], by a chain of products in fp64."""
    v = np.ones((M.shape[0], 1))
    for n, c in enumerate(cores):
        v = np.einsum("pa,apb->pb", v, np.asarray(c, dtype=np.float64)[:, M[:, n], :])
    return v.sum(axis=1)


class Problem:
    """The function and what it is sampled on: a grid (list of 1-D axes) or input TTs (lists of numpy cores)."""

    def __init__(self, function, domain=None, tensors=None, function_arg="vectors", minimize=False):
        assert (domain is None) != (tensors is None)
        self.function, self.function_arg, self.minimize = function, function_arg, minimize
        self.axes = None if domain is None else [np.asarray(a, dtype=np.float64) for a in domain]
        self.tensors = tensors
        self.Is = [len(a) for a in self.axes] if tensors is None else [c.shape[1] for c in tensors[0]]

    def coords(self, M):
        """The function's arguments at the multi-indices M [P, N]."""
        if self.tensors is None:
            return [self.axes[k][M[:, k]] for k in range(M.shape[1])]
        return [tt_values(t, M) for t in self.tensors]

    def __call__(self, xs):
        if self.function_arg == "matrix":
            y = np.asarray(self.function(np.stack(xs, axis=1)), dtype=np.float64)
        else:
            y = np.asarray(self.function(*xs), dtype=np.float64)
        return y[:, 0] if y.ndim == 2 else y


def fibres(lset, rset, I):
    """Multi-indices (a, i, c) -> (lset[a, 1:], i, rset[c, :-1]) in the reference's sample order [Rl * I * Rr, N]."""
    Rl, Rr = lset.shape[0], rset.shape[0]
    left = np.repeat(lset[:, 1:], I * Rr, axis=0)
    mid = np.tile(np.repeat(np.arange(I), Rr), Rl)[:, None]
    right = np.tile(rset[:, :-1], (Rl * I, 1))
    return np.concatenate([left, mid, right], axis=1).astype(np.int64)


class Step:
    """What one sweep step produced."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def evaluate(prob, lset, rset, j, state):
    """cross.py:316-379: the samples of core j ([Rl, I, Rr]) after the _minimize transform, with their coordinates."""
    I = prob.Is[j]
    M = fibres(lset, rset, I)
    xs = prob.coords(M)
    raw = prob(xs)
    vals = raw
    if prob.minimize:  # cross.py:342-359
        vals = np.pi / 2 - np.arctan(raw - state["min"])
        am = int(np.argmax(vals))
        emin = np.tan(np.pi / 2 - vals[am]) + state["min"]
        if state["min"] == 0 or emin < state["min"]:
            state["min"] = emin
            state["argmin"] = tuple(int(v) for v in M[am])
    state["nsamples"] += vals.size
    return M, xs, raw, vals.reshape(lset.shape[0], I, rset.shape[0])


def pick(prob, Q):
    if prob.minimize:  # cross.py:399-400: rect_maxvol(Q, maxK=r)
        return rect_maxvol(Q, maxK=Q.shape[1])
    return maxvol(Q)


def left_step(prob, lset, rset, j, state):
    """cross.py:391-420 for core j: samples -> QR -> maxvol -> core = Q inv(Q[local]) -> lsets[j + 1]."""
    M, xs, raw, V3 = evaluate(prob, lset, rset, j, state)
    Rl, I, Rr = V3.shape
    V = V3.reshape(Rl * I, Rr)
    Q = np.linalg.qr(V)[0]
    local, _, mv = pick(prob, Q)
    core = np.linalg.solve(Q[local].T, Q.T).T.reshape(Rl, I, Rr)
    local_r, local_i = np.divmod(np.asarray(local, dtype=np.int64), I)
    nxt = np.c_[lset[local_r, :], local_i]
    return Step(M=M, xs=xs, raw=raw, V=V, Q=Q, local=np.asarray(local), core=core, set=nxt, margin=mv["margin"], mv=mv,
                cond=_cond(V))


def _cond(V):
    s = np.linalg.svd(V, compute_uv=False)
    return float(s[-1] / s[0]) if s[0] > 0 else 0.0


def right_step(prob, lset, rset, j, state):
    """cross.py:423-451 for core j: samples -> QR of the transposed right unfolding -> maxvol -> core -> rsets[j - 1]."""
    M, xs, raw, V3 = evaluate(prob, lset, rset, j, state)
    Rl, I, Rr = V3.shape
    V = V3.reshape(Rl, I * Rr)
    Q = np.linalg.qr(V.T)[0]
    local, _, mv = pick(prob, Q)
    core = np.linalg.solve(Q[local].T, Q.T).reshape(Rl, I, Rr)
    local_i, local_r = np.divmod(np.asarray(local, dtype=np.int64), Rr)
    nxt = np.c_[local_i, rset[local_r, :]]
    return Step(M=M, xs=xs, raw=raw, V=V, Q=Q, local=np.asarray(local), core=core, set=nxt, margin=mv["margin"], mv=mv,
                cond=_cond(V))


def clamp_ranks(Rs, Is):
    Rs = np.array(Rs)
    N = len(Is)
    for n in list(range(1, N)) + list(range(N - 1, -1, -1)):
        Rs[n] = min(Rs[n - 1] * Is[n - 1], Rs[n], Is[n] * Rs[n + 1])
    return Rs


def run(prob, ranks_tt=None, kickrank=3, rmax=100, eps=1e-6, max_iter=25, val_size=1000, on_step=None):
    """The whole of cross.py:138-529 on `prob`, drawing from the global NumPy and torch RNGs exactly as cross.py does.
    on_step(kind, j, step, sets), if given, sees every step ('L' / 'R') and may return the index set to continue from
    (e.g. the device's), so a caller can restart each step from another implementation's state.
    Returns (cores, info) with the reference's info keys (Rs, nsamples, lsets, rsets, val_epss, val_eps, min, argmin)
    plus `margin` (the smallest decision margin met), `cond` (the smallest sample-matrix cond) and `steps`."""
    Is = prob.Is
    N = len(Is)
    if ranks_tt is None:
        ranks_tt = 1
    else:
        kickrank = None
    if not hasattr(ranks_tt, "__len__"):
        ranks_tt = [ranks_tt] * (N - 1)
    Rs = clamp_ranks([1] + list(ranks_tt) + [1], Is)
    for n in range(N):  # cross.py:277: the initial cores are drawn, never used
        torch.randn(int(Rs[n]), Is[n], int(Rs[n + 1]))
    lsets = [np.zeros((1, 1), dtype=np.int64)] + [None] * (N - 1)
    randint = np.hstack([np.random.randint(0, Is[n + 1], [max(Rs), 1]) for n in range(N - 1)]
                        + [np.zeros([max(Rs), 1], dtype=int)])
    rsets = [randint[: Rs[n + 1], n:] for n in range(N - 1)] + [np.zeros((1, 1), dtype=np.int64)]
    Mval = np.stack([np.random.choice(I, int(val_size)) for I in Is], axis=1)
    ys_val = prob(prob.coords(Mval))
    state = dict(nsamples=0, min=0, argmin=None)
    info = dict(val_epss=[], margin=np.inf, cond=np.inf, steps=0)
    cores = [None] * N
    val_eps = np.inf
    for it in range(max_iter):
        for j in range(N - 1):
            s = left_step(prob, lsets[j], rsets[j], j, state)
            info["margin"], info["cond"] = min(info["margin"], s.margin), min(info["cond"], s.cond)
            info["steps"] += 1
            cores[j] = s.core
            got = on_step("L", j, s, (lsets, rsets)) if on_step else None
            lsets[j + 1] = s.set if got is None else got
        for j in range(N - 1, 0, -1):
            s = right_step(prob, lsets[j], rsets[j], j, state)
            info["margin"], info["cond"] = min(info["margin"], s.margin), min(info["cond"], s.cond)
            info["steps"] += 1
            cores[j] = s.core
            got = on_step("R", j, s, (lsets, rsets)) if on_step else None
            rsets[j - 1] = s.set if got is None else got
        M, xs, raw, V3 = evaluate(prob, lsets[0], rsets[0], 0, state)
        cores[0] = V3
        if on_step:
            on_step("F", 0, Step(M=M, xs=xs, raw=raw, core=V3), (lsets, rsets))
        val_eps = float(np.linalg.norm(ys_val - tt_values(cores, Mval)) / np.linalg.norm(ys_val))
        info["val_epss"].append(val_eps)
        if val_eps < eps:
            break
        if it < max_iter - 1 and kickrank is not None:  # cross.py:481-498
            newRs = Rs.copy()
            newRs[1:-1] = np.minimum(rmax, newRs[1:-1] + kickrank)
            for n in list(range(1, N)) + list(range(N - 1, 0, -1)):
                newRs[n] = min(newRs[n - 1] * Is[n - 1], newRs[n], Is[n] * newRs[n + 1])
            extra = np.hstack([np.random.randint(0, Is[n + 1], [max(newRs), 1]) for n in range(N - 1)]
                              + [np.zeros([max(newRs), 1], dtype=int)])
            for n in range(N - 1):
                if newRs[n + 1] > Rs[n + 1]:
                    rsets[n] = np.vstack([rsets[n], extra[: newRs[n + 1] - Rs[n + 1], n:]])
            Rs = newRs
    info.update(Rs=Rs, nsamples=state["nsamples"], lsets=lsets, rsets=rsets, val_eps=val_eps, min=state["min"],
                argmin=state["argmin"], Mval=Mval)
    return cores, info


def run_batch(problems, ranks_tt, eps=1e-6, max_iter=25, val_size=1000):
    """cross_batch's contract: problem b equals the b-th of len(problems) sequential cross() runs from one RNG state."""
    return [run(p, ranks_tt=ranks_tt, eps=eps, max_iter=max_iter, val_size=val_size) for p in problems]
