"""`Tensor.__getitem__` with the reference's semantics (tntorch/tensor.py:1019-1434).

Key forms: integers (negative ones wrap), slices with steps, None, Ellipsis, index arrays (lists, tuples, NumPy arrays,
CPU or CUDA tensors) and a 2-D P x N matrix (one index array per column).  Index arrays must appear contiguously.

Results have the reference's type and core shapes (for TT and Tucker tensors):
- an all-integer key gives a 0-d tensor, from one P = 1 library call (ops.tt_gather);
- a run of index arrays (with the run of integers right before it) is one ops.tt_gather range call, the [r, P, r'] core
  the reference builds by multiplying core[:, idx, :] slices;
- any other run of integers is a P = 1 range call, joined into the next core (or, at the end, into the previous one);
- a slice keeps its core sliced (or, under a Tucker factor, the core whole and the factor sliced), None adds an
  identity core.
Tucker factors of integer and index modes are absorbed into their cores first; CP cores are turned into TT cores, so a
CP tensor gives the reference's values in TT cores.  On a batch tensor the first key entry indexes the batch: an integer
gives a non-batch result, a slice a batch one whose gathers are one ops.tt_gather_batch call each.  When a core or a
factor requires grad, the gathers of fp32 and fp64 cores stay library calls, differentiated by one tnb_tt_gather_grad
call each; Tucker absorption and the joins of integer runs are torch products then, so autograd reaches the factors
(and CP factors through _cp_to_tt).  Cores of any other dtype take the reference's torch chain under grad.
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops


def _kind(k) -> str:
    if hasattr(k, "__len__"):
        return "index"
    if k is None:
        return "none"
    if isinstance(k, (int, np.integer)):
        return "int"
    if isinstance(k, slice):
        return "slice"
    raise IndexError(f"unsupported index entry {k!r}")


def process_key(key, nmodes: int) -> list:
    """The key as one entry per mode (and None entries), the reference's _process_key (tensor.py:1019-1055)."""
    if isinstance(key, (torch.Tensor, np.ndarray)) and key.ndim == 2:
        key = [key[:, j] for j in range(key.shape[1])]
    if not hasattr(key, "__len__"):
        key = [key]
    elif isinstance(key, (torch.Tensor, np.ndarray)):
        key = [key]
    elif isinstance(key, tuple):
        key = list(key)
    elif any(not np.isscalar(k) for k in key):
        key = list(key)
    else:
        key = [key]  # a list of integers is one index array
    nonecount = sum(1 for k in key if k is None)
    for i, k in enumerate(key):
        if k is Ellipsis:
            key = key[:i] + [slice(None)] * (nmodes - (len(key) - nonecount) + 1) + key[i + 1:]
            break
    if any(k is Ellipsis for k in key):
        raise IndexError("Only one ellipsis is allowed, at most")
    if nmodes - (len(key) - nonecount) < 0:
        raise IndexError("Too many index entries {} vs {}".format(nmodes, len(key) - nonecount))
    return key + [slice(None)] * (nmodes - (len(key) - nonecount))


def _int_value(k, n: int) -> int:
    v = int(k)
    if not -n <= v < n:
        raise IndexError(f"index {v} is out of bounds for a mode of size {n}")
    return v + n if v < 0 else v


def _index_array(k, n: int, device) -> torch.Tensor:
    """An index array as an int64 tensor, negatives wrapped (as torch indexing wraps them); on the cores' device when it
    came as a CUDA tensor, on the host otherwise (ops.tt_gather checks the range where the key lives)."""
    if isinstance(k, torch.Tensor):
        a = k.detach().long()
        if a.is_cuda and a.device != device:
            a = a.to(device)
    else:
        a = torch.as_tensor(np.asarray(k)).long()
    if a.dim() != 1:
        raise IndexError("index arrays must be one-dimensional")
    return torch.where(a < 0, a + n, a)


class _View:
    """The tensor being indexed: TT cores (3-D, or 4-D with a leading batch dimension) and Tucker factors."""

    def __init__(self, cores, Us, batch):
        self.cores, self.Us, self.batch = cores, Us, batch
        self.grad = any(c.requires_grad for c in cores) or any(U is not None and U.requires_grad for U in Us)

    def n(self, k):
        return self.cores[k].shape[-2] if self.Us[k] is None else self.Us[k].shape[-2]

    # ---- products, batched over a leading dimension in batch mode
    def mm(self, A, B):
        """A [.., i, j] @ B [.., j, k] (per sample in batch mode)."""
        if self.grad:
            return A @ B
        if A.dim() == 2:
            return ops.matmul(A.contiguous(), B.contiguous())
        return torch.stack([ops.matmul(A[b].contiguous(), B[b].contiguous()) for b in range(A.shape[0])])

    def absorbed(self, k):
        """Core k with its Tucker factor absorbed ('ijk,aj->iak'), as the reference's get_key does for integer and
        index modes."""
        c, U = self.cores[k], self.Us[k]
        if U is None:
            return c
        r0, S, r1 = c.shape[-3:]
        lead = c.shape[:-3]
        m = self.mm(U, c.transpose(-3, -2).reshape(lead + (S, r0 * r1)))  # [.., I, r0 r1]
        return m.reshape(lead + (U.shape[-2], r0, r1)).transpose(-3, -2).contiguous()

    def gather(self, f, l, cols, P):
        """[.., r_f, P, r_l]: the product of the slices of modes f..l-1 at the P points `cols` (one index tensor per
        mode)."""
        cores = [self.absorbed(k) for k in range(f, l)]
        if self.grad and cores[0].dtype not in (torch.float32, torch.float64):
            # a dtype the library does not take: the reference's chain of core[:, idx, :] products (tensor.py:1286-1330)
            dev = cores[0].device
            s = cores[0][..., cols[0].to(dev), :]
            for c, ix in zip(cores[1:], cols[1:]):
                s = torch.einsum("...iaj,...jak->...iak", s, c[..., ix.to(dev), :])
            return s
        on_dev = any(c.is_cuda for c in cols)
        idx = torch.stack([c.to(cores[0].device) if on_dev else c for c in cols], dim=1)
        if self.batch:
            return ops.tt_gather_batch([[c[b] for c in cores] for b in range(cores[0].shape[0])], idx)
        return ops.tt_gather(cores, idx)


def getitem(t, key):
    from .tensor import Tensor

    if isinstance(key, Tensor):
        raise NotImplementedError("indexing by a mask Tensor needs the automata module, which is not built")
    if isinstance(key, torch.Tensor) and not key.is_cuda:
        key = key.detach().long()
    nd = t.dim()
    key = process_key(key, nd + (1 if t.batch else 0))

    cores, Us, batch = list(t.cores), list(t.Us), t.batch
    if any(c.dim() != (4 if batch else 3) for c in cores):  # CP factors become TT cores (values equal the reference's)
        tt = Tensor(cores, Us=Us, batch=batch)
        tt._cp_to_tt()
        cores = tt.cores
    if batch:
        k0, key = key[0], key[1:]
        kind0 = _kind(k0)
        if kind0 == "none":
            raise ValueError("Cannot change batch dimension")
        if kind0 == "index":
            raise ValueError("Advanced indexing is prohibited for batch dimension")
        if kind0 == "int":
            b = _int_value(k0, cores[0].shape[0])
            cores, Us, batch = [c[b] for c in cores], [None if U is None else U[b] for U in Us], False
        else:
            cores, Us = [c[k0] for c in cores], [None if U is None else U[k0] for U in Us]
    v = _View(cores, Us, batch)
    dev = cores[0].device

    out_cores, out_Us = [], []
    ints = []          # pending run of (mode, value)
    block = None       # pending index block: (first mode, [index tensors])
    block_done = False
    P = None

    def run_matrix(run):
        """The [.., r_f, r_l] product of a run of integer modes: one P = 1 range call."""
        f, l = run[0][0], run[-1][0] + 1
        cols = [torch.tensor([val], dtype=torch.int64) for _, val in run]
        m = v.gather(f, l, cols, 1)
        return m[..., :, 0, :]

    def emit(core, U=None):
        nonlocal ints
        if ints:
            m = run_matrix(ints)
            r0, a, r1 = core.shape[-3:]
            core = v.mm(m, core.reshape(core.shape[:-3] + (r0, a * r1))).reshape(core.shape[:-3] + (m.shape[-2], a, r1))
            ints = []
        out_cores.append(core)
        out_Us.append(U)

    def flush():
        nonlocal block, block_done, ints
        if block is None:
            return
        f, cols = block
        core = v.gather(f, f + len(cols), cols, P)
        out_cores.append(core)
        out_Us.append(None)
        block, block_done = None, True

    k = 0  # mode of the tensor
    for entry in key:
        kind = _kind(entry)
        if kind == "none":
            flush()
            r = cores[k].shape[-3] if k < nd else cores[-1].shape[-1]
            eye = torch.eye(r, dtype=cores[0].dtype, device=dev)[:, None, :]
            if batch:
                eye = eye.expand((cores[0].shape[0],) + eye.shape).clone()
            emit(eye)
            continue
        n = v.n(k)
        if kind == "slice":
            flush()
            if Us[k] is None:
                emit(cores[k][..., entry, :])
            else:
                emit(cores[k], Us[k][..., entry, :])
        elif kind == "int":
            flush()
            ints.append((k, _int_value(entry, n)))
        else:
            if block_done:
                raise IndexError("All index arrays must appear contiguously")
            a = _index_array(entry, n, dev)
            if block is None:
                P = a.shape[0]
                pre = [torch.full((P,), val, dtype=torch.int64, device=a.device) for _, val in ints]
                block = (ints[0][0] if ints else k, pre + [a])
                ints = []
            else:
                if a.shape[0] != P:
                    raise ValueError("Index arrays must have the same length")
                block[1].append(a)
        k += 1
    flush()
    if ints:
        m = run_matrix(ints)
        if not out_cores:  # every entry an integer: the value
            if not batch and m.numel() > 1:
                return torch.sum(m)
            return torch.squeeze(m)
        last = out_cores[-1]
        r0, a, r1 = last.shape[-3:]
        out_cores[-1] = v.mm(last.reshape(last.shape[:-3] + (r0 * a, r1)), m).reshape(
            last.shape[:-3] + (r0, a, m.shape[-1]))
    return Tensor(out_cores, Us=out_Us, batch=batch)
