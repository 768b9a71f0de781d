"""CPU restatement of tnb_tt_gather_grad (csrc/tt_gather_grad.cuh): the stable order of each mode's points, the chunks
of a mode's reduction, the path of each reverse step and reduction, the launches a call makes and the workspace it asks
for; and the fp64 NumPy backward in that order, chunk by chunk,
dG_k[:, i, :] = sum over the points with index i at mode k of L_k^T W_k."""
import numpy as np

import ttg_model as tm

SORT_CHUNK = 256 * 16
CHUNK_MIN, CHUNK_MAX, CHUNK_CTAS, BK = 256, 1 << 16, 1024, 32
# the kernel each branch runs, as a profiler trace names it
STEP_KERNELS = {tm.TC: "ttg_step_tc_kernel", tm.RANK_MIN: "ttg_step_generic_kernel",
                tm.RANK_MAX: "ttg_step_generic_kernel"}
REDUCE_KERNELS = {tm.TC: "ttgg_reduce_tc_kernel", tm.RANK_MIN: "ttgg_reduce_generic_kernel",
                  tm.RANK_MAX: "ttgg_reduce_generic_kernel"}


def _cdiv(a, b):
    return -(-a // b)


def sort_passes(n):
    p = 1
    while p < 4 and (n >> (8 * p)) > 0:
        p += 1
    return p


def chunk_rows(rows, rk, rk1):
    otiles = _cdiv(rk, tm.T) * _cdiv(rk1, 64)
    ch = _cdiv(_cdiv(rows * otiles, CHUNK_CTAS), BK) * BK
    return min(max(ch, CHUNK_MIN), CHUNK_MAX)


def chunk_bound(rows, n, ch):
    return _cdiv(rows, ch) + n + 1


def slot_bound(rows, ch):
    return 2 * rows // ch if rows > ch else 0


def buckets(idx, shape, first, last):
    """[M][P] bucket of every point at every mode: its index, or I_k for every mode of a point with any index out of
    range."""
    idx = np.asarray(idx, np.int64)
    n = np.array(shape[first:last])
    bad = ((idx < 0) | (idx >= n)).any(axis=1)
    return np.where(bad[None, :], n[:, None], idx.T)


def order(bucket):
    """The stable order of the points by bucket (the radix sort's)."""
    return np.argsort(bucket, kind="stable")


def chunks(bucket, n, ra, ch):
    """(value, first row, row count) of each chunk of a mode's reduction, in bucket order."""
    cnt = np.bincount(bucket, minlength=n + 1) * ra
    out, row = [], 0
    for b in range(n + 1):
        for q in range(_cdiv(int(cnt[b]), ch)):
            out.append((b, row + q * ch, min(ch, int(cnt[b]) - q * ch)))
        row += int(cnt[b])
    return out


def mode_paths(r, first, last):
    """The path of every mode's reduction (first .. last - 1) and reverse step (first + 1 .. last - 1)."""
    return [tm.mode_path(r[k], r[k + 1]) for k in range(first, last)]


def kernels(r, first, last):
    """The set of step and reduction kernel names one train's backward runs."""
    names = set()
    for k in range(first, last):
        p = tm.mode_path(r[k], r[k + 1])
        names.add(REDUCE_KERNELS[p])
        if k > first:
            names.add(STEP_KERNELS[p])
    return names


def launches(shape, ranks, first, last):
    M = last - first
    n = 1 + sum(1 + 3 * sort_passes(shape[k]) for k in range(first, last))
    per = (M - 1) + M + (M - 1 if M > 1 else 0) + 1 + 2 * M + (M - 1)
    return n + len(ranks) * per


def _align(x):
    return (x + 255) // 256 * 256


def workspace_bytes(shape, ranks, first, last, P, esize):
    M = last - first
    ncounts = sum(shape[k] + 1 for k in range(first, last))
    passes = max(sort_passes(shape[k]) for k in range(first, last))
    lsum_max = w_max = tiles_max = chunks_max = part_max = 0
    for r in ranks:
        rows = P * r[first]
        lsum = sum(rows * r[k] for k in range(first + 1, last))
        tl = sum(3 * tm.tile_bound(rows, shape[k]) + 1 for k in range(first + 1, last))
        cl = 0
        for k in range(first, last):
            ch = chunk_rows(rows, r[k], r[k + 1])
            cl += 4 * chunk_bound(rows, shape[k], ch) + 1
            part_max = max(part_max, slot_bound(rows, ch) * r[k] * r[k + 1])
        lsum_max, w_max = max(lsum_max, lsum), max(w_max, rows * max(r[first + 1:last + 1]))
        tiles_max, chunks_max = max(tiles_max, tl), max(chunks_max, cl)
    b = _align(P * M * 4) + _align(ncounts * 4) + _align(P * M * 4)
    if passes > 1:
        b += _align(P * 4)
    b += _align(256 * _cdiv(P, SORT_CHUNK) * 4)
    if tiles_max > 0:
        b += _align(tiles_max * 4)
    b += _align(chunks_max * 4)
    if lsum_max > 0:
        b += _align(lsum_max * esize)
    b += 2 * _align(w_max * esize)
    if part_max > 0:
        b += _align(part_max * esize)
    return max(b, 256)


def grad(cores, idx, grad_out, first=0, last=None, absolute=False):
    """The gradients of the range's cores in fp64 (of the chain in absolute values when `absolute`, for error bounds),
    summed as the device sums: per mode over chunks of the stable order, the chunks in order."""
    last = len(cores) if last is None else last
    f = (lambda c: np.abs(np.asarray(c, np.float64))) if absolute else (lambda c: np.asarray(c, np.float64))
    G = [f(c) for c in cores]
    shape = [c.shape[1] for c in cores]
    ranks = [G[0].shape[0]] + [c.shape[2] for c in G]
    ra, P, M = ranks[first], len(idx), last - first
    bk = buckets(idx, shape, first, last)
    ix = np.minimum(bk, np.array(shape[first:last])[:, None] - 1)  # excluded points address nothing that counts
    Ls = [None] * M
    s = G[first][:, ix[0], :]  # [ra, P, r]
    for m in range(1, M):
        Ls[m] = s
        s = np.einsum("apb,bpc->apc", s, G[first + m][:, ix[m], :])
    W = f(grad_out)  # [ra, P, r_last]
    out = [None] * M
    for m in range(M - 1, -1, -1):
        k = first + m
        n = shape[k]
        L = np.broadcast_to(np.eye(ra)[:, None, :], (ra, P, ra)) if m == 0 else Ls[m]
        Lr = L.transpose(1, 0, 2).reshape(P * ra, -1)  # rows (p, a)
        Wr = W.transpose(1, 0, 2).reshape(P * ra, -1)
        perm = order(bk[m])
        rows = (perm[:, None] * ra + np.arange(ra)[None, :]).reshape(-1)
        ch = chunk_rows(P * ra, ranks[k], ranks[k + 1])
        dG = np.zeros((ranks[k], n, ranks[k + 1]))
        for b, r0, c in chunks(bk[m], n, ra, ch):
            if b < n:
                rr = rows[r0:r0 + c]
                dG[:, b, :] += Lr[rr].T @ Wr[rr]
        out[m] = dG
        if m > 0:
            W = np.einsum("apc,bpc->apb", W, G[k][:, ix[m], :])
    return out
