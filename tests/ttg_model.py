"""CPU restatement of tnb_tt_gather's plan (csrc/tt_gather.cuh): the per-call path (ttg_path: fused or grouped), the
per-step path of the grouped modes (ttg_mode_path), the tile bound of a step, the launches a call makes and the
workspace it asks for; and the fp64 NumPy chain the device computes,
out[t][a][p][b] = (G_first[:, i_p0, :] ... G_{last-1}[:, i_p(M-1), :])[a, b]."""
import numpy as np

FUSED, GROUPED = range(2)
TC, RANK_MIN, RANK_MAX = range(3)
PATHS = {FUSED: "fused", GROUPED: "grouped"}
BRANCHES = {TC: "tensor cores", RANK_MIN: "a rank below 16", RANK_MAX: "a rank above 256"}
TC_MIN_R, TC_MAX_R = 16, 256
FUSED_MAX_ROWS, FUSED_MAX_STATE, FUSED_MAX_MODES = 4096, 2048, 64
T = 64  # state rows per tile
# the kernel each branch runs, as a profiler trace names it
PATH_KERNELS = {FUSED: "ttg_fused_kernel", GROUPED: "ttg_init_kernel"}
MODE_KERNELS = {TC: "ttg_step_tc_kernel", RANK_MIN: "ttg_step_generic_kernel", RANK_MAX: "ttg_step_generic_kernel"}


def _cdiv(a, b):
    return -(-a // b)


def _align(x):
    return (x + 255) // 256 * 256


def state_cols(r, first, last):
    return max([r[k] for k in range(first + 1, last)], default=0)


def path(ranks, first, last, P):
    """ranks: per-train rank profiles (lists of ndim + 1)."""
    if last - first > FUSED_MAX_MODES:
        return GROUPED
    for r in ranks:
        w = max([r[last]] + [r[k] for k in range(first + 1, last)])
        if P * r[first] > FUSED_MAX_ROWS or r[first] * w > FUSED_MAX_STATE:
            return GROUPED
    return FUSED


def mode_path(rk, rk1):
    if max(rk, rk1) > TC_MAX_R:
        return RANK_MAX
    if min(rk, rk1) < TC_MIN_R:
        return RANK_MIN
    return TC


def mode_paths(r, first, last):
    """The path of every grouped step (modes first + 1 .. last - 1) of one train."""
    return [mode_path(r[k], r[k + 1]) for k in range(first + 1, last)]


def tile_bound(rows, n):
    return _cdiv(rows, T) + n + 1


def launches(ranks, first, last, P):
    """Fused: one per train.  Grouped: one narrowing the indices, then per train one for the first mode and four per
    later mode (histogram, scan, scatter, step)."""
    if path(ranks, first, last, P) == FUSED:
        return len(ranks)
    return 1 + len(ranks) * (1 + 4 * (last - first - 1))


def workspace_bytes(shape, ranks, first, last, P, esize):
    if path(ranks, first, last, P) == FUSED:
        return 256
    M = last - first
    nmax = max(shape[first:last])
    rows_max = max(P * r[first] for r in ranks)
    state_max = max(P * r[first] * state_cols(r, first, last) for r in ranks)
    tiles_max = max([tile_bound(P * r[first], shape[k]) for r in ranks for k in range(first + 1, last)], default=0)
    b = _align(P * M * 4) + _align((nmax + 1) * 4)
    if M > 1:
        b += _align((nmax + 1) * 4) + _align((3 * tiles_max + 1) * 4) + _align(rows_max * 4)
    if state_max > 0:
        b += 2 * _align(state_max * esize)
    return max(b, 256)


def gather(cores, idx, first=0, last=None, absolute=False):
    """[r_first, P, r_last] in fp64 (of |G| when `absolute`: the chain in absolute values, for error bounds)."""
    last = len(cores) if last is None else last
    idx = np.asarray(idx)
    f = (lambda c: np.abs(np.asarray(c, np.float64))) if absolute else (lambda c: np.asarray(c, np.float64))
    s = f(cores[first])[:, idx[:, 0], :]
    for m, k in enumerate(range(first + 1, last), start=1):
        s = np.einsum("apb,bpc->apc", s, f(cores[k])[:, idx[:, m], :])
    return s


def depth(ranks, first, last):
    """K of the bound c K u (chain in absolute values): the terms a value's sums run over, along the chain."""
    return max(1, sum(ranks[k] for k in range(first + 1, last)))
