"""NumPy restatement of tnb_tt_hadamard_round (csrc/tt_hadamard_round.cuh): round_tt(a * b) from the left Grams of the
product and the Gram of each bond's carry, never forming the Kronecker cores.  Used by the CPU tests to check the method
against the fp64 oracle and the library's sizing and path choosers against their restatement."""
import math

import numpy as np

TC_MIN_R, TC_MAX_R = 16, 256
MAX_KEEP = 256
CHUNK_DOUBLES = 1 << 26
PATH_TC, PATH_RANK_MIN, PATH_RANK_MAX, PATH_FORCED = 0, 1, 2, 3


def mode_path(ra, rb, rao, rbo, allow_tc=True):
    """tthr_mode_path"""
    if not allow_tc:
        return PATH_FORCED
    lo, hi = min(ra, rb, rao, rbo), max(ra, rb, rao, rbo)
    if hi > TC_MAX_R:
        return PATH_RANK_MAX
    if lo < TC_MIN_R:
        return PATH_RANK_MIN
    return PATH_TC


def bond_path(n, k, allow_tc=True):
    """tthr_bond_path"""
    if not allow_tc:
        return PATH_FORCED
    return PATH_RANK_MIN if min(n, k) < TC_MIN_R else PATH_TC


def chunk(n, ra, rb, rao, rbo):
    """tthr_chunk: mode values per launch of the recurrence"""
    per = max(rb * ra * rb * rao, rb * rao * rbo * rao) + ra * rb * rao * rbo
    return max(1, min(CHUNK_DOUBLES // max(per, 1), n, 65535))


def dims(shape, ra, rb, rmax=None):
    """make_hr_dims: product ranks, rank caps, output slots and capacity."""
    N = len(shape)
    R = [a * b for a, b in zip(ra, rb)]
    rorth = [1] * (N + 1)
    for k in range(N - 1):
        rorth[k + 1] = min(rorth[k] * shape[k], R[k + 1])
    rm = [0] * max(N - 1, 0) if rmax is None else list(rmax)
    rcap = [1] * (N + 1)
    for mu in range(N - 1, 0, -1):
        c = min(rorth[mu], shape[mu] * rcap[mu + 1])
        if rm[mu - 1] > 0:
            c = min(c, rm[mu - 1])
        rcap[mu] = min(c, MAX_KEEP)
    slot, off = [], 0
    for k in range(N):
        slot.append(off)
        off += rcap[k] * shape[k] * rcap[k + 1]
        off = (off + 63) // 64 * 64
    return dict(R=R, rorth=rorth, rcap=rcap, slot=slot, capacity=off)


def gl_step(GL, A, B):
    """GL_{k+1} = sum_i (A_i (x) B_i)^T GL_k (A_i (x) B_i) as the four one-index contractions of the kernel."""
    ra, I, rao = A.shape
    rb, _, rbo = B.shape
    G = GL.reshape(ra, rb, ra, rb)
    out = np.zeros((rao, rbo, rao, rbo))
    for i in range(I):
        T1 = np.einsum("abcd,ax->bcdx", G, A[:, i, :])
        T2 = np.einsum("bcdx,by->cdxy", T1, B[:, i, :])
        T3 = np.einsum("cdxy,cz->dxyz", T2, A[:, i, :])
        out += np.einsum("dxyz,dw->xyzw", T3, B[:, i, :])
    return out.reshape(rao * rbo, rao * rbo)


def left_grams(a, b):
    N = len(a)
    GL = [np.ones((1, 1))]
    for k in range(N - 1):
        GL.append(gl_step(GL[k], a[k].astype(np.float64), b[k].astype(np.float64)))
    return GL


def carry(A, B, W):
    """Y = (A_mu (x) B_mu) W, [R_mu, I r'], B contracted first."""
    ra, I, rao = A.shape
    rb, _, rbo = B.shape
    rn = W.shape[1]
    Wt = W.reshape(rao, rbo, rn)
    Z = np.einsum("xyj,biy->ixjb", Wt, B)
    Y = np.einsum("aix,ixjb->abij", A, Z)
    return Y.reshape(ra * rb, I * rn)


def rank_rule(w, delta2, cap):
    """round.py:137-158 on descending eigenvalues (squared singular values): smallest rank whose tail is <= delta^2."""
    w = np.clip(w, 0, None)
    L = len(w)
    cum, count = 0.0, 0
    for i in range(L - 1, -1, -1):
        cum += w[i]
        if cum <= delta2:
            count += 1
        else:
            break
    return max(1, min(L - count, cap))


def hadamard_round(a, b, eps=1e-14, rmax=None):
    """(cores, ranks, norm_sq, discarded_sq) of round_tt(a * b) by the library's method, in fp64."""
    N = len(a)
    a = [np.asarray(c, dtype=np.float64) for c in a]
    b = [np.asarray(c, dtype=np.float64) for c in b]
    shape = [c.shape[1] for c in a]
    ra = [1] + [c.shape[2] for c in a]
    rb = [1] + [c.shape[2] for c in b]
    d = dims(shape, ra, rb, rmax)
    rm = [0] * max(N - 1, 0) if rmax is None else list(rmax)
    GL = left_grams(a, b)
    W = np.ones((1, 1))
    cores = [None] * N
    ranks = [1] * (N + 1)
    norm2, disc, delta2 = None, 0.0, 0.0
    for mu in range(N - 1, 0, -1):
        Y = carry(a[mu], b[mu], W)
        H = Y.T @ GL[mu] @ Y
        H = 0.5 * (H + H.T)
        tr = float(np.trace(H))
        if norm2 is None:
            norm2 = tr
            delta2 = (eps / max(1.0, math.sqrt(N - 1))) ** 2 * tr
        w, V = np.linalg.eigh(H)
        w, V = w[::-1], V[:, ::-1]
        n = H.shape[0]
        kcap = min(d["rcap"][mu], n)
        cap = min(n, rm[mu - 1]) if rm[mu - 1] > 0 else n
        zero = math.sqrt(max(w[0], 0.0)) < 1e-13
        r = 1 if zero else min(rank_rule(w, delta2, cap), kcap)
        disc += tr if zero else max(tr - float(np.clip(w[:r], 0, None).sum()), 0.0)
        Vr = np.zeros((n, 1)) if zero else V[:, :r]
        cores[mu] = Vr.T.reshape(r, shape[mu], ranks[mu + 1])
        W = Y @ Vr
        ranks[mu] = r
    Y = carry(a[0], b[0], W)
    cores[0] = Y.reshape(1, shape[0], ranks[1])
    if norm2 is None:
        norm2 = float((Y ** 2).sum())
    return cores, ranks, norm2, disc


def kronecker(a, b):
    """The product's Kronecker cores (Tensor.__mul__, tensor.py:560-640)."""
    out = []
    for A, B in zip(a, b):
        ra, I, rao = A.shape
        rb, _, rbo = B.shape
        out.append(np.einsum("aix,biy->abixy", A, B).reshape(ra * rb, I, rao * rbo))
    return out


def full(cores):
    t = np.ones((1, 1))
    for c in cores:
        t = np.einsum("pr,rix->pix", t, c).reshape(-1, c.shape[2])
    return t.reshape([c.shape[1] for c in cores])
