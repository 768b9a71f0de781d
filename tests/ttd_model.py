"""CPU restatement of tnb_tt_dot's plan (csrc/tt_dot.cuh): the association order and envelope of each mode of each pair
(ttd_order, ttd_mode_path), the split over i (ttd_chunks), the launches a call makes and the workspace it asks for; and
the fp64 NumPy chain F_{k+1} = sum_i A_k[:, i, :]^T F_k B_k[:, i, :] the device computes."""
import numpy as np

TC, RANK_MIN, RANK_MAX = range(3)
BRANCHES = {TC: "tensor cores", RANK_MIN: "a rank below 16", RANK_MAX: "a rank above 256"}
BM, GN, TARGET, GROUP = 32, 64, 512, 32


def _cdiv(a, b):
    return -(-a // b)


def order(ra, rb, rao, rbo):
    """True: B first."""
    return rbo * ra * (rb + rao) < rao * rb * (ra + rbo)


def mode_path(rx, ry, rxo, ryo):
    if max(rx, ry, rxo, ryo) > 256:
        return RANK_MAX
    if min(rx, ry, rxo, ryo) < 16:
        return RANK_MIN
    return TC


def plan(npairs, n, ra, rb, rao, rbo):
    """(swap, path, rxo, ryo, work items per chunk, chunks) of one mode of one pair."""
    swap = order(ra, rb, rao, rbo)
    rx, ry, rxo, ryo = (rb, ra, rbo, rao) if swap else (ra, rb, rao, rbo)
    path = mode_path(rx, ry, rxo, ryo)
    tiles = _cdiv(rxo, BM) * (1 if path == TC else _cdiv(ryo, GN))
    c = min(max(_cdiv(TARGET, npairs * tiles), 1), n)
    nch = _cdiv(n, _cdiv(n, c))
    return swap, path, rxo, ryo, tiles, nch


def paths(shape, ranks_a, ranks_b):
    """Per pair, the path of every mode; ranks_a / ranks_b are lists of per-pair rank profiles."""
    P = len(ranks_a)
    return [[plan(P, n, a[k], b[k], a[k + 1], b[k + 1])[1] for k, n in enumerate(shape)]
            for a, b in zip(ranks_a, ranks_b)]


def launches(shape, ranks_a, ranks_b):
    p = paths(shape, ranks_a, ranks_b)
    total = 0
    for k in range(len(shape)):
        for g0 in range(0, len(p), GROUP):
            used = {p[q][k] == TC for q in range(g0, min(g0 + GROUP, len(p)))}
            total += len(used) + 1
    return total


def _align(x):
    return (x + 255) // 256 * 256


def workspace_bytes(shape, ranks_a, ranks_b):
    P, N = len(ranks_a), len(shape)
    f = sum(max([a[k] * b[k] for k in range(1, N)], default=0) for a, b in zip(ranks_a, ranks_b))
    part = 0
    for k, n in enumerate(shape):
        s = 0
        for a, b in zip(ranks_a, ranks_b):
            _, _, rxo, ryo, _, nch = plan(P, n, a[k], b[k], a[k + 1], b[k + 1])
            s += nch * rxo * ryo
        part = max(part, s)
    return max((_align(f * 8) if f else 0) + _align(part * 8), 256)


def dot(a, b):
    """<a, b> of two trains of NumPy cores, the fp64 chain: per mode G = F^T A (rb x n ra'), then G^T B over (rb, n)."""
    f = np.ones((1, 1))
    for x, y in zip(a, b):
        x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
        ra, n, rao = x.shape
        rb, _, rbo = y.shape
        g = (f.T @ x.reshape(ra, n * rao)).reshape(rb * n, rao)
        f = g.T @ y.reshape(rb * n, rbo)
    return float(f[0, 0])


def tt_cores(cores, Us=None):
    """Plain TT cores of a TT / CP train with optional Tucker factors [I, S] (tensor.py:1576-1627, 1717-1762)."""
    out = []
    N = len(cores)
    for k, c in enumerate(cores):
        c = np.asarray(c, np.float64)
        U = None if Us is None else Us[k]
        if U is not None:
            c = U @ c if c.ndim == 2 else np.einsum("asb,is->aib", c, np.asarray(U, np.float64))
        if c.ndim == 2:  # CP factor [I, R]: diagonal slices
            I, R = c.shape
            if k == 0:
                c = c[None]
            elif k == N - 1:
                c = c.T[:, :, None]
            else:
                d = np.zeros((R, I, R))
                d[np.arange(R), :, np.arange(R)] = c.T
                c = d
        out.append(c)
    return out


def abs_dot(a, b):
    """<|a|, |b|>: the scale of the rounding error bound of <a, b>."""
    return dot([np.abs(np.asarray(x, np.float64)) for x in a], [np.abs(np.asarray(y, np.float64)) for y in b])


def depth(shape, ranks_a, ranks_b):
    """The longest chain of fp64 additions behind one F entry: per mode, n times (ra + rb)."""
    return sum(n * (max(ranks_a[k], 1) + max(ranks_b[k], 1)) for k, n in enumerate(shape))
