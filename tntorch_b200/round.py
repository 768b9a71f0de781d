"""Module-level mirrors of tntorch/round.py:7-187 (clone-then-round wrappers, truncated_svd)."""
from __future__ import annotations

import math
from typing import Optional

import torch

from . import ops


def round_tt(t, **kwargs):
    """round.py:7-19"""
    t2 = t.clone()
    t2.round_tt(**kwargs)
    return t2


def round_tucker(t, **kwargs):
    """round.py:22-34"""
    t2 = t.clone()
    t2.round_tucker(**kwargs)
    return t2


def round(t, **kwargs):
    """round.py:37-49"""
    t2 = t.clone()
    t2.round(**kwargs)
    return t2


def truncated_svd(
    M: torch.Tensor,
    delta: Optional[float] = None,
    eps: Optional[float] = None,
    rmax: Optional[int] = None,
    left_ortho: Optional[bool] = True,
    algorithm: Optional[str] = "svd",
    verbose: Optional[bool] = False,
    batch: Optional[bool] = False,
):
    """round.py:52-187.  `algorithm` is accepted for signature parity; both values run the same
    Gram + eigen kernels (the reference's own 'eig' formulation) with fp64 accumulation."""
    if delta is not None and eps is not None:
        raise ValueError("Provide either `delta` or `eps`")
    assert rmax is None or rmax >= 1
    assert algorithm in ("svd", "eig")
    if batch:
        # batch mode ignores eps/delta (round.py:149-150): rank = min(rmax, len(S))
        outs = [ops.truncated_svd(M[b], rmax=rmax, left_ortho=left_ortho, batch_mode=True, return_zero_flag=True)
                for b in range(M.shape[0])]
        if all(o[2] for o in outs):  # round.py:138-142: every sample is zero -> rank-1 zero factors
            return (torch.zeros(M.shape[0], M.shape[1], 1, dtype=M.dtype, device=M.device),
                    torch.zeros(M.shape[0], 1, M.shape[2], dtype=M.dtype, device=M.device))
        return torch.stack([o[0] for o in outs]), torch.stack([o[1] for o in outs])
    return ops.truncated_svd(M, delta=delta, eps=eps, rmax=rmax, left_ortho=left_ortho)


def reduce(ts, function, eps=0, rmax=None, algorithm="svd", verbose=False, **kwargs):
    """tools.py:460-512: a function of all tensors of a sequence, climbing a binary tree and rounding every intermediate.
    For `operator.add` (and `operator.sub`'s accumulate form) the node `tn.round(a + b)` is ONE library call
    (tnb_tt_sum_round: block cores assembled in the workspace, then the rounding sweeps).  For `operator.mul` the node
    `tn.round(a * b)` is one tnb_tt_hadamard_round call when the Kronecker cores cannot be rounded (a product rank above
    256, or not enough device memory: ops.hadamard_round_instead_of_kronecker), and runs as before otherwise.  Any other
    function is applied as given and rounded with `round`."""
    import operator

    from .tensor import Tensor

    assert algorithm in ("svd", "eig")
    fused = function is operator.add and not kwargs
    product = function is operator.mul and not kwargs

    def node(a, b):
        if fused and not a.batch and not b.batch:
            return Tensor(ops.tt_sum_round([a._tt_cores(), b._tt_cores()], eps=eps, rmax=rmax))
        if product and isinstance(a, Tensor) and isinstance(b, Tensor) and not a.batch and not b.batch:
            out = _hadamard_round_node(a, b, eps, rmax, algorithm)
            if out is not None:
                return out
        out = function(a, b, **kwargs)
        out.round(eps=eps, rmax=rmax, algorithm=algorithm)
        return out

    d = dict()
    for elem in ts:
        climb = 0
        while climb in d:
            elem = node(d[climb], elem)
            d.pop(climb)
            climb += 1
        d[climb] = elem
    keys = list(d.keys())
    result = d[keys[0]]
    for key in keys[1:]:
        result = node(result, d[key])
    return result


def _hadamard_round_node(a, b, eps, rmax, algorithm):
    """`round(a * b, eps, rmax)` as reduce's `operator.mul` node takes it when the Kronecker path cannot run
    (ops.hadamard_round_instead_of_kronecker): one fused tt_hadamard_round call, then Tensor.round's Tucker step with the
    left-over budget, the error reached taken from the returned energies.  None: the Kronecker path runs as before."""
    from .tensor import Tensor

    c0 = a.cores[0]
    if c0.dtype != b.cores[0].dtype or list(a.shape) != list(b.shape):
        return None
    # the TT ranks _tt_cores() would give (a CP tensor's boundary ranks are 1), read without converting anything
    ra, rb = [int(r) for r in a.ranks_tt], [int(r) for r in b.ranks_tt]
    ra[0] = ra[-1] = rb[0] = rb[-1] = 1
    free, _ = torch.cuda.mem_get_info(c0.device)
    if not ops.hadamard_round_instead_of_kronecker(list(a.shape), ra, rb, c0.element_size(), int(free)):
        return None
    ca, cb = a._tt_cores(), b._tt_cores()
    cores, info = ops.tt_hadamard_round(ca, cb, eps=eps, rmax=rmax, return_info=True)
    out = Tensor(cores)
    nn = info["norm_sq"]
    reached = math.sqrt(info["discarded_sq"] / nn) if nn > 0 else 0.0
    if reached < eps:
        out.round_tucker((1 + eps) / (1 + reached) - 1, rmax=rmax, algorithm=algorithm)
    return out


def relative_error(gt, approx):
    """metrics.py:135-151.  (dense torch tensor, Tensor): one device reconstruct-and-diff call.  (Tensor, Tensor): both
    are decompressed as before when their dense tensors fit in free device memory; otherwise (ops.dot_instead_of_dense)
    the reference's formula on three TT dots from one call, sqrt(max(<g, g> + <a, a> - 2 <g, a>, 0) / max(<g, g>, 0)),
    which cannot resolve errors below about 1e-8."""
    from .tensor import Tensor

    if isinstance(gt, torch.Tensor) and isinstance(approx, Tensor) and not approx.batch and all(c.dim() == 3 for c in approx.cores):
        if any(U is not None for U in approx.Us):
            approx = approx.decompress_tucker_factors()
        return ops.tt_relative_error(gt.to(approx.cores[0].device), approx.cores)
    if isinstance(gt, Tensor) and isinstance(approx, Tensor) and not gt.batch and not approx.batch:
        dense = math.prod(gt.shape) * gt.cores[0].element_size() + math.prod(approx.shape) * approx.cores[0].element_size()
        free, _ = torch.cuda.mem_get_info(gt.cores[0].device)
        if ops.dot_instead_of_dense(dense, int(free)):
            a, b = gt._tt_cores(), approx._tt_cores()
            gg, aa, ga = ops.tt_dot_batch([(a, a), (b, b), (a, b)])
            return float(torch.sqrt((gg + aa - 2 * ga).clamp(0)) / torch.sqrt(gg.clamp(0)))
    a = gt.torch() if isinstance(gt, Tensor) else gt
    b = approx.torch() if isinstance(approx, Tensor) else approx
    return float(torch.dist(a, b) / torch.norm(a))
