"""Host-side mirror of the reference's `tn.Tensor` for the decomposition / rounding path.

Same constructor signature, attribute names and error behaviour as rballester/tntorch
(tntorch/tensor.py:107-439), restricted to the hot path this package accelerates:
dense -> TT (``ranks_tt=`` / ``eps=``), TT cores in / out, ``round_tt``, ``round``, ``torch()``.
Everything numerical runs in libtnb200.so on the GPU; there is no CPU path.
"""
from __future__ import annotations

import contextlib
from typing import Any, Optional, Sequence, Union

import numpy as np
import torch

from . import ops


def _default_device(device):
    if device is None:
        if not torch.cuda.is_available():
            raise RuntimeError("tntorch_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        return torch.device("cuda", torch.cuda.current_device())
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError(f"tntorch_b200 runs on CUDA devices only, got device={device}")
    return device


def _streams(data: torch.Tensor, ranks_tt, dev) -> bool:
    """Whether a rank-capped decomposition of `data` streams it from host memory (ops.ttsvd_stream) instead of copying
    it to `dev`: only for a CPU tensor of two or more modes whose device image plus the device call's workspace exceeds
    free device memory (ops.stream_instead_of_copy)."""
    if data.is_cuda or data.dim() < 2:
        return False
    shape = list(data.shape)
    sh, rm, _, _ = ops._ttsvd_layout(shape, ranks_tt)
    wsb = ops.lib().tnb_ttsvd_workspace_bytes(ops._dense_code(data.dtype), len(shape), sh, rm, 0)
    free, _ = torch.cuda.mem_get_info(dev)
    return ops.stream_instead_of_copy(data.numel() * data.element_size(), int(wsb), int(free))


class Tensor(object):
    """TT tensor whose decomposition / rounding runs on H100 kernels (mirror of tntorch.Tensor)."""

    def __init__(
        self,
        data: Union[torch.Tensor, np.ndarray, Sequence[torch.Tensor]],
        Us: Optional[Union[torch.Tensor, Any]] = None,
        idxs: Optional[Any] = None,
        device: Optional[Any] = None,
        requires_grad: Optional[bool] = None,
        ranks_cp: int = None,
        ranks_tucker: Optional[Sequence[int]] = None,
        ranks_tt: Optional[Sequence[int]] = None,
        eps: Optional[float] = None,
        max_iter: Optional[int] = 25,
        tol: Optional[float] = 1e-4,
        verbose: Optional[bool] = False,
        batch: Optional[bool] = False,
        algorithm: Optional[str] = "svd",
    ):
        assert algorithm in ("svd", "eig")  # both map onto the same Gram/eigen kernels
        self.batch = batch
        if isinstance(data, (list, tuple)):  # explicit cores (tensor.py:163-192)
            min_dim, max_dim = (3, 4) if batch else (2, 3)
            if not all(min_dim <= d.dim() <= max_dim for d in data):
                raise ValueError("All tensor cores must have 2 (for CP) or 3 (for TT) dimensions")
            d1, d2 = (1, 2) if batch else (0, 1)
            for n in range(len(data) - 1):  # tensor.py:177-191
                if (data[n + 1].dim() == max_dim and data[n].shape[-1] != data[n + 1].shape[d1]) or (
                    data[n + 1].dim() == min_dim and data[n].shape[-1] != data[n + 1].shape[d2]
                ):
                    raise ValueError("Core ranks do not match")
            dev = _default_device(device if device is not None else (data[0].device if data[0].is_cuda else None))
            self.cores = [c.to(dev) for c in data]
            N = len(data)
        else:
            if isinstance(data, np.ndarray):
                data = torch.as_tensor(data)
            elif not isinstance(data, torch.Tensor):
                raise ValueError(
                    "A tntorch.Tensor may be built either from a list of cores, one NumPy ndarray, or one PyTorch tensor"
                )
            dev = _default_device(device if device is not None else (data.device if data.is_cuda else None))
            stream = (ranks_tt is not None and eps is None and ranks_cp is None and ranks_tucker is None and not batch
                      and _streams(data, ranks_tt, dev))
            if not stream:
                data = data.to(dev)
            if data.dim() == 0:
                if data.dtype in (torch.float8_e4m3fn, torch.float8_e5m2):  # torch has no arithmetic on float8
                    data = data.reshape(1).clone()
                else:
                    data = data * torch.ones(1, device=dev, dtype=data.dtype)
            if eps is not None and ranks_tt is not None:
                raise ValueError("Specify eps or ranks, but not both")  # tensor.py:436-438
            N = data.dim() - 1 if batch else data.dim()
            if ranks_cp is not None:  # CP-ALS (tensor.py:210-400)
                if ranks_tt is not None:
                    raise ValueError("ALS for CP-TT is not yet supported")
                assert not hasattr(ranks_cp, "__len__")
                if eps is not None:
                    raise ValueError("Specify eps or ranks, but not both")
                if ranks_tucker is not None:
                    # CP on Tucker's core (tensor.py:278-302): exact TT -> round_tucker(rmax=ranks_tucker) -> the dense
                    # Tucker core -> ALS from RANDOM factors (torch.randn, like the reference); the Tucker factors stay
                    if batch:
                        raise NotImplementedError("batched CP on a Tucker core is not built")
                    self.cores = ops.ttsvd(data, rmax=None, eps=0.0)
                    self.Us = [None] * N
                    self.round_tucker(rmax=ranks_tucker, algorithm=algorithm)
                    core = self.tucker_core().contiguous()
                    init = [torch.randn(sh, ranks_cp, dtype=core.dtype, device=dev) for sh in core.shape]
                    self.cores = ops.cp_als(core, ranks_cp, max_iter=max_iter, tol=tol, init=init)
                    Us = self.Us
                elif batch:
                    self.cores = [torch.stack(f, dim=0) for f in zip(*[
                        ops.cp_als(data[b], ranks_cp, max_iter=max_iter, tol=tol) for b in range(data.shape[0])])]
                else:
                    self.cores = ops.cp_als(data, ranks_cp, max_iter=max_iter, tol=tol)
            elif eps is not None and ranks_tucker is None and not batch:
                # tensor.py:436-439: _full_rank_tt + round(eps) = round_tt(eps) then round_tucker with the left-over
                # budget.  The exact TT is never formed: the dense sweep with the eps rank rule IS _full_rank_tt +
                # round_tt(eps), and `reached` (tensor.py:2096, error of the rounded TT against the exact one) is the
                # error against the dense data, measured by the device reconstruct-and-diff kernel.
                self.cores = ops.ttsvd(data, rmax=None, eps=eps)
                self.Us = [None] * N
                # a 1-mode "tensor" is stored exactly by its single core: nothing to measure (and the error kernel needs N >= 2)
                reached = float(ops.tt_relative_error(data, self.cores)) if N >= 2 else 0.0
                if reached < eps:
                    self.round_tucker((1 + eps) / (1 + reached) - 1, algorithm=algorithm)
                Us = self.Us
            elif ranks_tucker is not None:
                # tensor.py:401-408: exact TT first (the reference's _full_rank_tt), then round_tucker / round_tt on it.
                # The exact TT needs every Gram of the sweep to fit the direct eigensolver.
                if batch:
                    raise NotImplementedError("batched Tucker rounding is not built")
                if eps is not None:
                    raise ValueError("Specify eps or ranks, but not both")
                self.cores = ops.ttsvd(data, rmax=None, eps=0.0)
                self.Us = [None] * N
                self.round_tucker(rmax=ranks_tucker, algorithm=algorithm)
                if ranks_tt is not None:
                    self.round_tt(rmax=ranks_tt, algorithm=algorithm)
                Us = self.Us
            elif batch:
                # the reference's batch mode: per-sample decomposition, rank = min(rmax, len(S)), no eps
                # one library call for the whole batch: several samples in flight inside libtnb200 (tnb_ttsvd_batch)
                per = ops.ttsvd_batch(data, rmax=ranks_tt, batch_mode=True)
                self.cores = [torch.stack([p[k] for p in per], dim=0) for k in range(N)]
            elif stream:
                with torch.cuda.device(dev):
                    self.cores = ops.ttsvd_stream(data, rmax=ranks_tt)
            else:
                self.cores = ops.ttsvd(data, rmax=ranks_tt)
        if Us is None:
            Us = [None] * N
        self.Us = Us
        if requires_grad:
            for c in self.cores:
                c.requires_grad_()
        if idxs is None:
            idxs = [torch.arange(sh, device=self.cores[0].device) for sh in self.shape]
        self.idxs = idxs

    # ------------------------------------------------------------------ structure
    def dim(self):
        return len(self.cores)

    @property
    def shape(self):
        return torch.Size([(self.Us[n].shape[-2] if self.Us[n] is not None else c.shape[-2])
                           for n, c in enumerate(self.cores)])

    @property
    def ranks_tucker(self):
        return torch.tensor([c.shape[-2] for c in self.cores])

    def tucker_core(self):
        """tensor.py:1565-1574"""
        return Tensor(self.cores, batch=self.batch).torch()

    def decompress_tucker_factors(self):
        """tensor.py:1576-1627: absorb every Tucker factor into its core (einsum 'ijk,aj->iak')."""
        cores = []
        for c, U in zip(self.cores, self.Us):
            if U is None:
                cores.append(c)
            elif c.dim() == 2:  # CP factor [S, R] under a Tucker factor [I, S]
                cores.append(ops.matmul(U, c.contiguous()))
            else:
                r0, S, r1 = c.shape
                m = ops.matmul(U, c.permute(1, 0, 2).reshape(S, r0 * r1))  # [I, r0*r1]
                cores.append(m.reshape(U.shape[0], r0, r1).permute(1, 0, 2).contiguous())
        return Tensor(cores, batch=self.batch)

    @property
    def ranks_tt(self):
        d1 = 1 if self.batch else 0
        first = self.cores[0].shape[d1] if self.cores[0].dim() == (4 if self.batch else 3) else self.cores[0].shape[-1]
        return torch.tensor([first] + [c.shape[-1] for c in self.cores])

    def numcoef(self):
        return sum(c.numel() for c in self.cores)

    def clone(self):
        return Tensor([c.clone() for c in self.cores], Us=[None if U is None else U.clone() for U in self.Us],
                      batch=self.batch)

    def __repr__(self):
        return f"{self.dim()}D TT tensor (H100): shape {list(self.shape)}, TT ranks {self.ranks_tt.tolist()}"

    # ------------------------------------------------------------------ arithmetic that feeds the rounding path
    def _tt_cores(self):
        """This tensor as plain TT cores (Tucker factors absorbed, CP factors turned into diagonal-slice cores)."""
        if self.batch:
            raise NotImplementedError("arithmetic on batched tensors is not built")
        t = self.decompress_tucker_factors() if any(U is not None for U in self.Us) else self
        if any(c.dim() != 3 for c in t.cores):
            t = Tensor([c for c in t.cores])
            t._cp_to_tt()
        return t.cores

    def __add__(self, other):
        """tensor.py:445-520 for TT operands: block cores (libtnb200 tnb_tt_sum); a scalar is added as a rank-1 term."""
        if isinstance(other, (int, float)):
            c0 = self.cores[0]
            ones = [torch.ones(1, s, 1, dtype=c0.dtype, device=c0.device) for s in self.shape]
            return Tensor(ops.tt_sum([self._tt_cores(), ones], alpha=[1.0, float(other)]))
        return Tensor(ops.tt_sum([self._tt_cores(), other._tt_cores()]))

    __radd__ = __add__

    def __sub__(self, other):
        if isinstance(other, (int, float)):
            return self + (-other)
        return Tensor(ops.tt_sum([self._tt_cores(), other._tt_cores()], alpha=[1.0, -1.0]))

    def __rsub__(self, other):
        return (-self) + other

    def __neg__(self):
        return self * -1.0

    def __mul__(self, other):
        """scalar: the first core is scaled (like the reference); tensor: elementwise product = Kronecker cores
        (tensor.py:560-640, libtnb200 tnb_tt_hadamard)."""
        if isinstance(other, (int, float)):
            cores = [c.clone() for c in self.cores]
            cores[0] = cores[0] * other
            return Tensor(cores, Us=[None if U is None else U.clone() for U in self.Us], batch=self.batch)
        return Tensor(ops.tt_hadamard(self._tt_cores(), other._tt_cores()))

    __rmul__ = __mul__

    def __truediv__(self, other):
        if isinstance(other, (int, float)):
            return self * (1.0 / other)
        raise NotImplementedError("tensor / tensor needs cross-approximation (tn.cross)")

    # ------------------------------------------------------------------ decompression (tensor.py:1639-1687)
    def torch(self, dtype=None, out=None):
        """The dense tensor.  With `dtype=` and/or `out=` it is written by one library call (ops.tt_decompress): float32
        cores to float32, bfloat16 or float16, float64 cores to float64, into `out` when given."""
        if dtype is not None or out is not None:
            return self._decompress(dtype, out)
        if self.batch:
            return torch.stack([Tensor([c[b] for c in self.cores]).torch() for b in range(self.cores[0].shape[0])])
        if any(U is not None for U in self.Us):
            return self.decompress_tucker_factors().torch()
        c0 = self.cores[0]
        r0 = c0.shape[0] if c0.dim() == 3 else c0.shape[1]
        f = torch.ones(1, r0, dtype=c0.dtype, device=c0.device)
        last = len(self.cores) - 1
        for n, c in enumerate(self.cores):  # tensor.py:1666-1680
            if c.dim() == 2:  # CP factor [I, R]
                if n < last:
                    f = torch.einsum("ai,bi->abi", f, c)
                else:
                    f = torch.einsum("ai,bi->ab", f, c)[..., None]
            elif c.requires_grad or f.requires_grad:  # differentiable path (cross_forward, tensor.py:1666-1680)
                f = torch.einsum("ai,ibj->abj", f, c)
            else:  # TT core: one library GEMM per core (tnb_matmul), no eager einsum
                f = ops.matmul(f.contiguous(), c.reshape(c.shape[0], -1)).reshape(-1, c.shape[-1])
            f = f.reshape(-1, f.shape[-1])
        f = f.sum(dim=-1) if f.shape[-1] > 1 else f[..., 0]
        return f.reshape(list(self.shape))

    def _decompress(self, dtype, out):
        """torch(dtype=, out=): plain TT cores through ops.tt_decompress; Tucker factors are absorbed first, a batch is
        one call per sample into the slices of the result."""
        if any(U is not None for U in self.Us):
            return self.decompress_tucker_factors()._decompress(dtype, out)
        if any(c.dim() != (4 if self.batch else 3) for c in self.cores):
            raise ValueError("torch(dtype=, out=) needs TT cores; CP factors decompress through torch() without arguments")
        if self.batch:
            B, c0 = self.cores[0].shape[0], self.cores[0]
            if out is None:
                out = torch.empty([B] + list(self.shape), dtype=c0.dtype if dtype is None else dtype, device=c0.device)
            elif out.shape[0] != B or not out.is_contiguous():
                raise ValueError(f"torch(out=): out must be contiguous with a leading batch dimension of {B}")
            for b in range(B):
                ops.tt_decompress([c[b] for c in self.cores], dtype=dtype, out=out[b])
            return out
        return ops.tt_decompress(self.cores, dtype=dtype, out=out)

    def numpy(self):
        return self.torch().detach().cpu().numpy()

    # ------------------------------------------------------------------ CP -> TT (tensor.py:1717-1762)
    def _cp_to_tt(self, factor=None):
        """Turn CP factors ([I, R], or [B, I, R] in a batch) into TT cores whose slices are diagonal matrices; the first
        / last factor become [1, I, R] / [R, I, 1] (tensor.py:1717-1762).  Pure layout: no arithmetic."""
        m = 3 if self.batch else 2
        if factor is None:
            if self.cores[0].dim() == m:
                self.cores[0] = self.cores[0][:, None, ...] if self.batch else self.cores[0][None, ...]
            for mu in range(1, self.dim() - 1):
                self.cores[mu] = self._cp_to_tt(self.cores[mu])
            if self.cores[-1].dim() == m:
                self.cores[-1] = self.cores[-1].transpose(-1, -2)[..., None].contiguous()
            return
        if factor.dim() == m + 1:  # already a TT core
            return factor
        R, I = factor.shape[-1], factor.shape[-2]
        idx = torch.arange(R, device=factor.device)
        if self.batch:
            core = torch.zeros(factor.shape[0], R, I, R, dtype=factor.dtype, device=factor.device)
            core[:, idx, :, idx] = factor.permute(2, 0, 1)  # advanced indices first: [R, B, I]
        else:
            core = torch.zeros(R, I, R, dtype=factor.dtype, device=factor.device)
            core[idx, :, idx] = factor.t()
        return core

    # ------------------------------------------------------------------ orthogonalisation (tensor.py:1764-1909)
    def _samples(self):
        """(number of samples, accessor) so that batched and plain tensors share one code path: the device kernels take
        one problem per call or a leading batch dimension (tnb_qr_householder)."""
        return self.cores[0].shape[0] if self.batch else 1

    def factor_orthogonalize(self, mu: int):
        """Pushes the Tucker factor's non-orthogonal part into its core (tensor.py:1771-1798): Us[mu] = Q R (device
        Householder QR), core <- core x_mode R (library GEMM)."""
        if self.Us[mu] is None:
            return
        U = self.Us[mu]
        Q, R = ops.qr(U, return_r=True)  # batched when U is [B, I, S]
        Q, R = Q.to(U.dtype), R.to(U.dtype)
        self.Us[mu] = Q
        c = self.cores[mu]
        cp = c.dim() == (3 if self.batch else 2)

        def push(core, Rm):  # core [r0, S, r1] (or CP [S, R]) with S contracted against Rm [a, S]
            if cp:
                return ops.matmul(Rm, core)                                        # [a, R]
            r0, S, r1 = core.shape
            out = ops.matmul(Rm, core.permute(1, 0, 2).reshape(S, r0 * r1))        # [a, r0 r1]
            return out.reshape(Rm.shape[0], r0, r1).permute(1, 0, 2).contiguous()

        if self.batch:
            self.cores[mu] = torch.stack([push(c[b], R[b]) for b in range(c.shape[0])])
        else:
            self.cores[mu] = push(c, R)

    def left_orthogonalize(self, mu: int):
        """Makes the mu-th core left-orthogonal and pushes the R factor to its right core; returns R
        (tensor.py:1800-1833).  Householder QR and the R push run in libtnb200 (tnb_qr_householder, tnb_matmul);
        CP factors are turned into TT cores first, like in the reference."""
        assert 0 <= mu < self.dim() - 1
        self.factor_orthogonalize(mu)
        nd = 4 if self.batch else 3
        if self.cores[mu].dim() != nd or self.cores[mu + 1].dim() != nd:
            self._cp_to_tt()
        c = self.cores[mu]
        nxt = self.cores[mu + 1]
        if self.batch:
            B = c.shape[0]
            Q, R = ops.qr(c.reshape(B, -1, c.shape[-1]), return_r=True)  # one batched launch
            Q, R = Q.to(c.dtype), R.to(c.dtype)
            self.cores[mu] = Q.reshape(c.shape[:-1] + (Q.shape[2],))
            self.cores[mu + 1] = torch.stack([ops.matmul(R[b], nxt[b].reshape(nxt.shape[1], -1)) for b in range(B)]).reshape(
                (B, R.shape[1]) + nxt.shape[2:])
            return R
        Q, R = ops.qr(c.reshape(-1, c.shape[-1]), return_r=True)
        Q, R = Q.to(c.dtype), R.to(c.dtype)
        self.cores[mu] = Q.reshape(c.shape[:-1] + (Q.shape[1],))
        self.cores[mu + 1] = ops.matmul(R, nxt.reshape(nxt.shape[0], -1)).reshape((R.shape[0],) + nxt.shape[1:])
        return R

    def right_orthogonalize(self, mu: int):
        """Makes the mu-th core right-orthogonal and pushes the L factor to its left core; returns L
        (tensor.py:1835-1879)."""
        assert 1 <= mu < self.dim()
        self.factor_orthogonalize(mu)
        nd = 4 if self.batch else 3
        if self.cores[mu].dim() != nd or self.cores[mu - 1].dim() != nd:
            self._cp_to_tt()
        c = self.cores[mu]
        prv = self.cores[mu - 1]
        if self.batch:
            B = c.shape[0]
            Q, L = ops.qr(c.reshape(B, c.shape[1], -1).transpose(1, 2).contiguous(), return_r=True)
            L, Q = L.transpose(1, 2).contiguous().to(c.dtype), Q.transpose(1, 2).contiguous().to(c.dtype)
            self.cores[mu] = Q.reshape((B, Q.shape[1]) + c.shape[2:])
            self.cores[mu - 1] = torch.stack([ops.matmul(prv[b].reshape(-1, prv.shape[-1]), L[b]) for b in range(B)]).reshape(
                prv.shape[:-1] + (L.shape[2],))
            return L
        Q, L = ops.qr(c.reshape(c.shape[0], -1).t().contiguous(), return_r=True)
        L, Q = L.t().contiguous().to(c.dtype), Q.t().contiguous().to(c.dtype)
        self.cores[mu] = Q.reshape((Q.shape[0],) + c.shape[1:])
        self.cores[mu - 1] = ops.matmul(prv.reshape(-1, prv.shape[-1]), L).reshape(prv.shape[:-1] + (L.shape[1],))
        return L

    def orthogonalize(self, mu: int):
        """All left and right orthogonalisations needed to make the tensor mu-orthogonal; returns (R, L)
        (tensor.py:1881-1909).  CP cores become TT cores first."""
        if mu < 0:
            mu += self.dim()
        self._cp_to_tt()
        dt, dev = self.cores[0].dtype, self.cores[0].device
        lead = (self.cores[0].shape[0],) if self.batch else ()
        R = torch.ones(lead + (1, 1), dtype=dt, device=dev)
        L = torch.ones(lead + (1, 1), dtype=dt, device=dev)
        for i in range(mu):
            R = self.left_orthogonalize(i)
        for i in range(self.dim() - 1, mu, -1):
            L = self.right_orthogonalize(i)
        return R, L

    # ------------------------------------------------------------------ rounding (tensor.py:2008-2098)
    @contextlib.contextmanager
    def _unchanged_on_error(self):
        """A rounding that raises part way (a refused eigensolve) leaves the tensor as it was: the rounding steps only
        rebind entries of `cores` / `Us`, never write into a tensor, so the lists of the start are put back."""
        cores, Us = list(self.cores), list(self.Us)
        try:
            yield
        except BaseException:
            self.cores, self.Us = cores, Us
            raise

    def round_tt(self, eps: float = 1e-14, rmax=None, algorithm: Optional[str] = "svd", verbose: Optional[bool] = False):
        """In place, by rebinding ``self.cores`` (same contract as the reference)."""
        assert algorithm in ("svd", "eig")
        N = self.dim()
        if not hasattr(rmax, "__len__"):
            rmax = [rmax] * (N - 1)
        assert len(rmax) == N - 1
        with self._unchanged_on_error():
            self._round_tt(eps, rmax)

    def _round_tt(self, eps, rmax):
        N = self.dim()
        self._cp_to_tt()  # tensor.py:2031: CP (or CP-Tucker) cores become TT (or TT-Tucker) ones
        for mu in range(N):  # orthogonalize() in the reference pushes the factors' non-orthogonal parts into the cores
            self.factor_orthogonalize(mu)
        if self.batch:
            B = self.cores[0].shape[0]
            per = ops.tt_round_batch([[c[b] for c in self.cores] for b in range(B)], eps=eps, rmax=rmax, batch_mode=True)
            self.cores = [torch.stack([p[k] for p in per], dim=0) for k in range(N)]
        else:
            self.cores = ops.tt_round(self.cores, eps=eps, rmax=rmax)

    def round_tucker(self, eps: float = 1e-14, rmax=None, dim="all", algorithm: Optional[str] = "svd"):
        """tensor.py:1911-2006, composed from the device primitives: orthogonalise to the last core, then for
        mu = N-1..0 push the core's non-orthogonality into the Tucker factor (Householder QR), split the factor with
        truncated_svd(left_ortho=True) under the budget eps/sqrt(len(dim)), absorb the remainder into the core and
        right-orthogonalise."""
        assert algorithm in ("svd", "eig")
        if self.batch:
            raise NotImplementedError("batched Tucker rounding is not built")
        N = self.dim()
        if not hasattr(rmax, "__len__"):
            rmax = [rmax] * N
        assert len(rmax) == N
        if dim == "all":
            dim = range(N)
        if not hasattr(dim, "__len__"):
            dim = [dim] * N
        with self._unchanged_on_error():
            self._round_tucker(eps, rmax, dim)

    def _round_tucker(self, eps, rmax, dim):
        N = self.dim()
        self.orthogonalize(-1)
        for mu in range(N - 1, -1, -1):
            c = self.cores[mu]
            r0, S, r1 = c.shape
            if self.Us[mu] is None:
                self.Us[mu] = torch.eye(S, dtype=c.dtype, device=c.device)
            Q, R = ops.qr(c.permute(0, 2, 1).reshape(r0 * r1, S), return_r=True)  # tensor.py:1972-1979
            Q, R = Q.to(c.dtype), R.to(c.dtype)
            k = Q.shape[1]
            self.Us[mu] = ops.matmul(self.Us[mu], R.t().contiguous())              # I x k
            left, right = ops.truncated_svd(self.Us[mu], eps=eps / (len(dim) ** 0.5), rmax=rmax[mu], left_ortho=True)
            self.Us[mu] = left                                                    # I x r
            newc = ops.matmul(Q, right.t().contiguous())                          # (r0 r1) x r
            self.cores[mu] = newc.reshape(r0, r1, -1).permute(0, 2, 1).contiguous()
            if mu > 0:
                self.right_orthogonalize(mu)

    def __getitem__(self, key):
        """tensor.py:1019-1434: NumPy-style indexing (see getitem.py); index arrays and integers are read by
        ops.tt_gather without forming core[:, idx, :]."""
        from .getitem import getitem

        return getitem(self, key)

    def _tt_dot(self, other):
        """<self, other> for two TT(-Tucker, -CP) tensors (metrics.dot) as a 0-d float64 tensor: one library call
        (ops.tt_dot) on the cores `_tt_cores()` gives."""
        return ops.tt_dot(self._tt_cores(), other._tt_cores())

    def dot(self, other, **kwargs):
        """tensor.py:2104-2109: see callers.dot."""
        from .callers import dot

        return dot(self, other, **kwargs)

    def norm(self):
        """tensor.py:2139-2144: see callers.norm."""
        from .callers import norm

        return norm(self)

    def normsq(self):
        """tensor.py:2146-2151: see callers.normsq."""
        from .callers import normsq

        return normsq(self)

    def round(self, eps: float = 1e-14, **kwargs):
        """tensor.py:2085-2098: TT rounding, then Tucker rounding with the left-over error budget."""
        copy = self.clone()
        with self._unchanged_on_error():
            self.round_tt(eps, **kwargs)
            a, b = copy._tt_cores(), self._tt_cores()
            aa, bb, ab = ops.tt_dot_batch([(a, a), (b, b), (a, b)])  # the three dots of metrics.relative_error, one call
            d = (aa + bb - 2 * ab).clamp(min=0)
            reached = float(torch.sqrt(d) / torch.sqrt(aa.clamp(min=0)))
            if reached < eps:
                kw = {k: v for k, v in kwargs.items() if k in ("rmax", "algorithm")}
                self.round_tucker((1 + eps) / (1 + reached) - 1, **kw)
