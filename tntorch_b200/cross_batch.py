"""Batched TT-cross: B independent black-box functions on ONE tensor-product grid with ONE rank profile, all sweeps
advanced together (BASELINE.json config 5: "Batched (B=512) TT-cross approximation of 32^6 black-box fn").

The reference rejects batches (cross.py:256-258): B problems are B sequential `tn.cross` calls, each with a device->host
copy + NumPy maxvol + lstsq per core.  Here one sweep step of ALL problems is
    gather the sample coordinates (tnb_cross_gather_coords)  ->  evaluate the function(s)  ->  one batched Householder
    QR (tnb_qr_householder)  ->  one batched maxvol (tnb_maxvol: index sets + interpolation cores)  ->  nested index
    sets updated on the device (tnb_cross_update_lsets / _rsets),
and the validation error of every problem comes from one kernel (tnb_cross_tt_eval).  Nothing is copied to the host
inside a sweep except the B validation errors that decide convergence.

Per problem the arithmetic, the sampling order of the global NumPy / torch RNGs and the stopping rule are those of
`tntorch_b200.cross.cross` with fixed ranks (ranks_tt given, no kickrank growth), i.e. those of the reference: problem b
of `cross_batch` equals the b-th of B sequential `cross` calls started from the same RNG state
(tests/test_gpu_cross.py::test_cross_batch_matches_sequential).
"""
from __future__ import annotations

import time

import numpy as np
import torch

from . import ops
from .tensor import Tensor


def cross_batch(functions, domain, ranks_tt, batch=None, eps=1e-6, max_iter=25, val_size=1000, function_arg="vectors",
                batched_function=False, return_info=False, device=None):
    """
    :param functions: a sequence of B callables f_b(*xs) (xs = N coordinate vectors), or — with batched_function=True —
        ONE callable f(pid, *xs) evaluated for all problems at once (pid: int64 problem index of every sample)
    :param domain: list of N 1-D coordinate vectors (the grid shared by the problems)
    :param ranks_tt: int or list of N-1 ints (fixed ranks: the reference's `ranks_tt=` mode, kickrank disabled)
    :param batch: B (required with batched_function=True)
    :return: a batch `Tensor` (cores [B, r, I, r']) and, with return_info, a dict with per-problem `val_eps`, `nsamples`,
        `iterations`, `lsets`, `rsets`
    """
    assert function_arg in ("vectors", "matrix")
    if batched_function:
        assert batch is not None, "pass batch=B with a batched function"
        B = int(batch)
    else:
        functions = list(functions)
        B = len(functions)
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device())
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("tntorch_b200.cross_batch runs on CUDA devices only")
    axes = [torch.as_tensor(a, dtype=torch.float64).to(device) for a in domain]
    Is = [int(a.numel()) for a in axes]
    N = len(Is)
    Imax = max(Is)
    grid = torch.zeros(N, Imax, dtype=torch.float64, device=device)
    for k, a in enumerate(axes):
        grid[k, : Is[k]] = a
    if not hasattr(ranks_tt, "__len__"):
        ranks_tt = [ranks_tt] * (N - 1)
    Rs = np.array([1] + list(ranks_tt) + [1])
    for n in list(range(1, N)) + list(range(N - 1, -1, -1)):  # feasibility clamp, cross.py:268-270
        Rs[n] = min(Rs[n - 1] * Is[n - 1], Rs[n], Is[n] * Rs[n + 1])
    Rs = [int(r) for r in Rs]
    start = time.time()

    def call(pid, xs):
        """values of every problem's function at its own samples: xs are N vectors of length B * P (problem-major)."""
        if function_arg == "matrix":
            args = [torch.stack(xs, dim=1)]
        else:
            args = list(xs)
        if batched_function:
            out = functions(pid, *args)
        else:
            P = xs[0].numel() // B
            out = torch.cat([functions[b](*[a[b * P: (b + 1) * P] for a in args]) for b in range(B)])
        if out.dim() == 2:
            out = out[:, 0]
        bad = torch.isnan(out) | torch.isinf(out)
        if bool(bad.any()):  # cross.py:361-375
            k0 = int(torch.nonzero(bad)[0].item())
            raise ValueError("Invalid return value for function of problem {}: f({}) = {}".format(
                int(pid[k0]), ", ".join("{:g}".format(float(x[k0])) for x in xs), float(out[k0])))
        return out.to(torch.float64)

    # ---- per problem, in order, the RNG draws a sequential cross() would make (cross.py:277-291) ----
    rsets_h = [np.zeros((B, Rs[n + 1], N - n - 1), dtype=np.int32) for n in range(N - 1)]
    val_h = np.zeros((B, int(val_size), N), dtype=np.int32)
    for b in range(B):
        for n in range(N):
            torch.randn(Rs[n], Is[n], Rs[n + 1])  # the reference's initial cores: drawn (RNG parity), never used
        randint = np.hstack([np.random.randint(0, Is[n + 1], [max(Rs), 1]) for n in range(N - 1)]
                            + [np.zeros([max(Rs), 1], dtype=int)])
        for n in range(N - 1):
            rsets_h[n][b] = randint[: Rs[n + 1], n: N - 1]
        for k in range(N):
            val_h[b, :, k] = np.random.choice(Is[k], int(val_size))
    lsets = [torch.zeros(B, 1, 0, dtype=torch.int32, device=device)] + [None] * (N - 1)
    rsets = [torch.as_tensor(r, device=device) for r in rsets_h] + [torch.zeros(B, 1, 0, dtype=torch.int32, device=device)]
    val_idx = torch.as_tensor(val_h, device=device)
    pid_val = torch.arange(B, device=device).repeat_interleave(int(val_size))
    xs_val = [axes[k][val_idx[:, :, k].reshape(-1).long()] for k in range(N)]
    ys_val = call(pid_val, xs_val).reshape(B, int(val_size))
    norm_ys_val = torch.linalg.vector_norm(ys_val, dim=1)

    cores = [torch.zeros(B, Rs[n], Is[n], Rs[n + 1], dtype=torch.float64, device=device) for n in range(N)]
    active = torch.ones(B, dtype=torch.int32, device=device)  # 0: converged, frozen (the sequential call would have returned)
    iterations = torch.zeros(B, dtype=torch.int64, device=device)
    nsamples = torch.zeros(B, dtype=torch.int64, device=device)
    val_eps = torch.full((B,), float("inf"), dtype=torch.float64, device=device)
    pid_cache = {}

    def evaluate(j):
        Rl, I, Rr = Rs[j], Is[j], Rs[j + 1]
        xs = ops.cross_gather_coords(lsets[j], rsets[j], grid, N, j, I)  # N vectors of length B * Rl * I * Rr
        P = Rl * I * Rr
        if P not in pid_cache:
            pid_cache[P] = torch.arange(B, device=device).repeat_interleave(P)
        V = call(pid_cache[P], xs).reshape(B, Rl, I, Rr)
        nsamples.add_(active.long() * P)
        return V

    def keep(new, old):
        """frozen problems keep their previous values"""
        if old is None:
            return new
        m = active.bool().reshape((B,) + (1,) * (new.dim() - 1))
        return torch.where(m, new, old)

    for it in range(max_iter):
        # ---- left-to-right (cross.py:391-420) ----
        for j in range(N - 1):
            V = evaluate(j).reshape(B, Rs[j] * Is[j], Rs[j + 1])
            Q = ops.qr(V)
            local, C = ops.maxvol(Q)  # batched: local int32 [B, R_{j+1}], C = Q inv(Q[local]) [B, R_j I_j, R_{j+1}]
            cores[j] = keep(C.reshape(B, Rs[j], Is[j], Rs[j + 1]), cores[j])
            lsets[j + 1] = ops.cross_update_lsets(lsets[j], local, Is[j], active if it > 0 else None, lsets[j + 1])
        # ---- right-to-left (cross.py:423-451) ----
        for j in range(N - 1, 0, -1):
            V = evaluate(j).reshape(B, Rs[j], Is[j] * Rs[j + 1])
            Q = ops.qr(V.transpose(1, 2).contiguous())
            local, C = ops.maxvol(Q)
            cores[j] = keep(C.transpose(1, 2).reshape(B, Rs[j], Is[j], Rs[j + 1]), cores[j])
            rsets[j - 1] = ops.cross_update_rsets(rsets[j], local, Rs[j + 1], active if it > 0 else None, rsets[j - 1])
        cores[0] = keep(evaluate(0), cores[0])  # cross.py:454-455
        approx = ops.cross_tt_eval(cores, val_idx)  # [B, val_size]
        ve = torch.linalg.vector_norm(ys_val - approx, dim=1) / norm_ys_val
        val_eps = torch.where(active.bool(), ve, val_eps)
        iterations.add_(active.long())
        # cross.py:460-462: a converged problem stops.  Written as "not below eps" so that a NaN val_eps (the unscaled
        # norm of a function beyond ~1e+-154 over- or underflows) keeps sweeping, as the sequential call does
        active = active * (~(val_eps < eps)).int()
        if not bool(active.any()) or it == max_iter - 1:
            break

    t = Tensor([c for c in cores], batch=True)
    if return_info:
        info = {"val_eps": val_eps, "nsamples": nsamples, "iterations": iterations, "Rs": np.array(Rs),
                "lsets": lsets, "rsets": rsets, "total_time": time.time() - start}
        return t, info
    return t
