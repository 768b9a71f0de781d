"""Callers of the rounding path that re-round in loops (SURVEY.md §8(f)-3), on the device entry points:

  dot           metrics.py:28-116     <a, b> through the small interface matrices, one library call (tnb_tt_dot)
  normsq, norm  metrics.py:298-319    <t, t> and its square root
  dist          metrics.py:119-132    ||t1 - t2|| from three dots in one call
  hadamard_sum  metrics.py:321-450    sum of the elementwise product of K tensors, re-rounding the running product
  shift_mode    tools.py:650-697      move one mode through a TT, one truncated_svd per position
  TTMatrix      matrix.py:12-140      matrix -> d-way (i_k x o_k) tensor -> TT-SVD (plain or batched)
  tt_multiply   matrix.py:420-443     X @ M for a TTMatrix M, one library call that never forms M

Only the parts that sit on the hot path are mirrored (construction, decompression, the product with a batch, the
re-rounding loops); the rest of the TT-matrix algebra (trace, det, inv, cholesky, CPMatrix) stays out of scope
(DESIGN.md §7)."""
from __future__ import annotations

import math
from typing import List, Sequence, Union

import numpy as np
import torch

from . import ops
from .tensor import Tensor


def _trains(t: Tensor):
    """The plain TT cores of `t`, one list per sample of a batch=True tensor."""
    if not t.batch:
        return [t._tt_cores()]
    if any(U is not None for U in t.Us) or any(c.dim() != 4 for c in t.cores):
        raise NotImplementedError("dot products of batched Tucker or CP tensors are not supported")
    return [[c[b] for c in t.cores] for b in range(t.cores[0].shape[0])]


def _check_pair(t1: Tensor, t2: Tensor, k=None):
    if k is not None:
        raise NotImplementedError("tn.dot: partial contractions (k=) are not supported")
    if t1.dim() != t2.dim():
        raise NotImplementedError(f"tn.dot: tensors of unequal dimension ({t1.dim()} and {t2.dim()}) are not supported")
    if t1.batch != t2.batch:
        raise NotImplementedError("tn.dot: a batched tensor with a plain one is not supported")
    if not np.array_equal(t1.shape, t2.shape):  # metrics.py:75-80
        raise ValueError("Dot product requires leading dimensions to be equal, but they are {} and {}".format(
            t1.shape, t2.shape))


def _dots(*pairs):
    """<t1, t2> for several pairs from one library call (ops.tt_dot_batch): a 0-d float64 tensor per pair, or a [B]
    one when the pair is batched (one dot per sample)."""
    spec, flat = [], []
    for t1, t2 in pairs:
        a = _trains(t1)
        b = a if t2 is t1 else _trains(t2)
        if len(a) != len(b):
            raise ValueError(f"tn.dot: batch sizes differ ({len(a)} and {len(b)})")
        spec.append((len(flat), len(a), t1.batch))
        flat += list(zip(a, b))
    out = ops.tt_dot_batch(flat)
    return [out[s:s + n] if batch else out[s] for s, n, batch in spec]


def dot(t1: Tensor, t2: Tensor, k=None):
    """metrics.dot (k = None) for two TT(-Tucker, -CP) tensors of the same shape: a 0-d float64 tensor, or [B] for
    batch=True tensors, from one library call (tnb_tt_dot, fp64 on the device).  k= and tensors of unequal dimension
    raise NotImplementedError; a shape mismatch raises ValueError like the reference."""
    _check_pair(t1, t2, k)
    return _dots((t1, t2))[0]


def normsq(t: Tensor):
    """metrics.normsq: <t, t>."""
    return dot(t, t)


def norm(t: Tensor):
    """metrics.norm: sqrt(max(<t, t>, 0))."""
    return torch.sqrt(torch.clamp(normsq(t), min=0))


def dist(t1: Tensor, t2: Tensor):
    """metrics.dist for two TT tensors: sqrt(<t1, t1> + <t2, t2> - 2 max(<t1, t2>, 0)), the three dots from one call.
    Like the reference's, this cannot resolve distances below about 1e-8 of the norms (the squares cancel)."""
    _check_pair(t1, t2)
    aa, bb, ab = _dots((t1, t1), (t2, t2), (t1, t2))
    return torch.sqrt(aa + bb - 2 * ab.clamp(0))


def _sum_all(cores: Sequence[torch.Tensor]):
    """Sum of every entry of a TT: each core is summed over its mode, the r x r' matrices are chained (fp64)."""
    f = torch.ones(1, cores[0].shape[0], dtype=torch.float64, device=cores[0].device)
    for c in cores:
        f = f @ c.sum(dim=1, dtype=torch.float64)
    return f.sum()


def _hadamard_sum_exact(cs: List[List[torch.Tensor]]):
    """The K-way interface tensor E[r_1..r_K] carried from the left: per mode, every operand's core is applied to its
    own axis for all mode values at once, then the mode is summed away (metrics.py:399-417)."""
    K, N = len(cs), len(cs[0])
    dev = cs[0][0].device
    E = torch.ones([1] * K, dtype=torch.float64, device=dev)
    for n in range(N):
        I = cs[0][n].shape[1]
        T = E[None].expand(I, *E.shape)
        for k in range(K):
            c = cs[k][n].double().permute(1, 0, 2)          # [I, r, r']
            T = T.movedim(k + 1, -1)                        # axis k last
            sh = T.shape
            T = torch.bmm(T.reshape(I, -1, sh[-1]), c).reshape(*sh[:-1], c.shape[-1]).movedim(-1, k + 1)
        E = T.sum(dim=0)
    return E.reshape(-1)[0]


def hadamard_sum(ts: Sequence[Tensor], algorithm: str = "exact", eps: float = None):
    """Sum over all entries of t_1 * t_2 * ... * t_K (metrics.hadamard_sum).

    'exact' contracts the K trains directly (cost grows with the product of the ranks).  'svd' / 'eig' keep a running
    product P <- round_tt(P * t_k, eps/sqrt(K-1)): Kronecker cores (tnb_tt_hadamard) followed by the rounding sweeps
    (tnb_tt_round), or one fused tnb_tt_hadamard_round call where those cannot run (a product rank above 256, or not
    enough device memory), so the interface never exceeds the rounded rank times r_k; the result is within eps * ||prod|| *
    sqrt(numel) of the exact sum (the reference re-rounds the same intermediate quantities mode by mode)."""
    assert algorithm in ("svd", "eig", "exact")
    assert all(list(ts[0].shape) == list(t.shape) for t in ts[1:])
    if any(t.batch for t in ts):
        raise ValueError("Batched tensors are not supported.")
    cs = [t._tt_cores() for t in ts]
    if algorithm == "exact" or len(ts) == 1:
        return float(_hadamard_sum_exact(cs))
    step_eps = (1e-14 if eps is None else eps) / math.sqrt(len(ts) - 1)
    P = cs[0]
    for k in range(1, len(cs)):
        P = _round_product(P, cs[k], step_eps)
    return float(_sum_all(P))


def _round_product(a, b, eps):
    """round_tt(a * b, eps) of two lists of TT cores: Kronecker cores and tt_round where they can run, else one fused
    tt_hadamard_round call (ops.hadamard_round_instead_of_kronecker)."""
    if a[0].dtype == b[0].dtype:
        shape = [c.shape[1] for c in a]
        ra = [a[0].shape[0]] + [c.shape[2] for c in a]
        rb = [b[0].shape[0]] + [c.shape[2] for c in b]
        free, _ = torch.cuda.mem_get_info(a[0].device)
        if ops.hadamard_round_instead_of_kronecker(shape, ra, rb, a[0].element_size(), int(free)):
            return ops.tt_hadamard_round(a, b, eps=eps)
    return ops.tt_round(ops.tt_hadamard(a, b), eps=eps)


def shift_mode(t: Tensor, n: int, shift: int, eps: Union[float, str] = 1e-3):
    """Move mode n by `shift` positions inside the train, in place (tools.shift_mode): orthogonalise at n, then per
    position merge the two neighbouring cores with swapped modes (library GEMM) and split them again with
    truncated_svd; eps='same' keeps every rank no larger than it was."""
    N = t.dim()
    assert 0 <= n + shift < N
    if shift == 0:
        return t
    if t.batch:
        raise ValueError("Batched tensors are not supported.")
    if any(U is not None for U in t.Us):
        d = t.decompress_tucker_factors()
        t.cores, t.Us = d.cores, [None] * N
    t.orthogonalize(n)
    cores = t.cores
    sign = 1 if shift > 0 else -1
    for i in range(n, n + shift, sign):
        c1, c2, left_ortho = (i, i + 1, True) if sign == 1 else (i - 1, i, False)
        R1, I1, R2 = cores[c1].shape
        _, I2, R3 = cores[c2].shape
        sc = ops.matmul(cores[c1].reshape(R1 * I1, R2), cores[c2].reshape(R2, I2 * R3))
        sc = sc.reshape(R1, I1, I2, R3).permute(0, 2, 1, 3).reshape(R1 * I2, I1 * R3).contiguous()
        if isinstance(eps, str):
            if eps != "same":
                raise ValueError("Relative error '{}' not recognized".format(eps))
            left, right = ops.truncated_svd(sc, eps=0, rmax=R2, left_ortho=left_ortho)
        elif eps >= 0:
            left, right = ops.truncated_svd(sc, eps=eps / math.sqrt(abs(shift)), left_ortho=left_ortho)
        else:
            raise ValueError("Relative error '{}' not recognized".format(eps))
        r = left.shape[1]
        cores[c1] = left.reshape(R1, I2, r)
        cores[c2] = right.reshape(r, I1, R3)
    return t


class TTMatrix:
    """A matrix of shape (prod i_k) x (prod o_k) stored as TT cores [r_k, i_k, o_k, r_{k+1}] (matrix.py:12-140):
    the matrix is viewed as the d-way tensor with modes (i_k o_k) and sent through the dense -> TT path
    (`Tensor(..., ranks_tt=ranks)`, batched through tnb_ttsvd_batch when a leading batch dimension is present)."""

    def __init__(self, t, ranks: List[int], input_dims: List[int], output_dims: List[int]):
        assert len(input_dims) == len(output_dims) and len(input_dims) > 0
        assert isinstance(ranks, list) and len(ranks) == len(input_dims) - 1
        self.input_dims = torch.tensor(input_dims)
        self.output_dims = torch.tensor(output_dims)
        self.d = d = len(input_dims)
        if isinstance(t, list):
            assert t[0].dim() in (4, 5)
            self.batch = t[0].dim() == 5
            self.cores = t
            self.ranks = torch.tensor([c.shape[-1] for c in t[:-1]])
            return
        M = t
        assert M.dim() in (2, 3)
        self.batch = M.dim() == 3
        assert math.prod(input_dims) == M.shape[-2] and math.prod(output_dims) == M.shape[-1]
        lead = [M.shape[0]] if self.batch else []
        off = len(lead)
        X = M.reshape(lead + list(input_dims) + list(output_dims))
        order = list(range(off)) + [off + k + s * d for k in range(d) for s in (0, 1)]     # i_0 o_0 i_1 o_1 ...
        X = X.permute(order).reshape(lead + [input_dims[k] * output_dims[k] for k in range(d)]).contiguous()
        tt = Tensor(X, ranks_tt=ranks, batch=self.batch)
        self.ranks = tt.ranks_tt[1:-1]
        self.cores = [c.reshape(*c.shape[: off + 1], input_dims[k], output_dims[k], c.shape[-1]) for k, c in enumerate(tt.cores)]

    def torch(self, dtype=None):
        """Back to the dense 2-D (or batched 3-D) matrix (matrix.py:120-160); with `dtype=` the TT part is one library
        call that writes that dtype (Tensor.torch(dtype=))."""
        d, off = self.d, 1 if self.batch else 0
        cores = [c.reshape(*c.shape[: off + 1], -1, c.shape[-1]) for c in self.cores]
        X = Tensor(cores, batch=self.batch).torch(dtype=dtype)
        idims, odims = self.input_dims.tolist(), self.output_dims.tolist()
        lead = [X.shape[0]] if self.batch else []
        X = X.reshape(lead + [s for k in range(d) for s in (idims[k], odims[k])])
        order = list(range(off)) + [off + 2 * k for k in range(d)] + [off + 2 * k + 1 for k in range(d)]
        return X.permute(order).reshape(lead + [math.prod(idims), math.prod(odims)])

    def numpy(self):
        return self.torch().detach().cpu().numpy()


def _tt_multiply_einsum(tt_matrix: TTMatrix, tensor: torch.Tensor) -> torch.Tensor:
    """The reference's chain (matrix.py:432-443): X.T, then one einsum per core.  The differentiable path."""
    idims = tt_matrix.input_dims.tolist()
    b = tensor.reshape(-1, math.prod(idims)).shape[0]
    result = tensor.reshape(b, -1).T.reshape(idims[0], -1)
    result = torch.einsum("id,lior->ldor", result, tt_matrix.cores[0])
    for k in range(1, tt_matrix.d):
        result = result.reshape(idims[k], -1, tt_matrix.cores[k].shape[0])
        result = torch.einsum("idr,riob->dob", result, tt_matrix.cores[k])
    return result.reshape(b, -1)


def tt_multiply(tt_matrix: TTMatrix, tensor: torch.Tensor) -> torch.Tensor:
    """tntorch.tt_multiply (matrix.py:420-443): `tensor` viewed as [b, I] times the TT-matrix, a fresh [b, O] tensor in
    the cores' dtype.  On the device (ops.tt_multiply, tnb_tt_multiply) unless `tensor` or a core requires grad, which
    runs the reference's einsum chain in torch so that autograd sees it."""
    assert len(tensor.shape) > 1
    if tt_matrix.batch:
        raise NotImplementedError("tt_multiply: batched TT-matrices are not supported")
    if tensor.requires_grad or any(c.requires_grad for c in tt_matrix.cores):
        return _tt_multiply_einsum(tt_matrix, tensor)
    return ops.tt_multiply(tt_matrix.cores, tensor)
