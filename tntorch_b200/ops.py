"""Thin torch-tensor wrappers over the C-ABI (device pointers in, torch tensors out).

PyTorch is plumbing here: device memory (caching allocator), the current stream and
``torch.distributed``.  All arithmetic happens inside libtnb200.so.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import check, i32, i64, lib

_DT = {torch.float32: _lib.TNB_F32, torch.float64: _lib.TNB_F64}


def _dtype_code(t: torch.Tensor) -> int:
    if t.dtype not in _DT:
        raise ValueError(f"tntorch_b200 supports float32/float64 tensors, got {t.dtype}")
    return _DT[t.dtype]


# The dense TT-SVD (ttsvd, ttsvd_batch, their plans, tt_relative_error) also reads bfloat16, float16 and float8 (e4m3fn,
# e5m2) data; its cores are float32.
_DT_F8 = {torch.float8_e4m3fn: _lib.TNB_F8E4M3, torch.float8_e5m2: _lib.TNB_F8E5M2}
_DT_DENSE = {**_DT, torch.bfloat16: _lib.TNB_BF16, torch.float16: _lib.TNB_F16, **_DT_F8}
_DT_LOW = (torch.bfloat16, torch.float16, *_DT_F8)  # read as they are, float32 cores


def _dense_code(dtype: torch.dtype) -> int:
    if dtype not in _DT_DENSE:
        raise ValueError("the dense TT-SVD supports float32/float64/bfloat16/float16/float8_e4m3fn/float8_e5m2 tensors, "
                         f"got {dtype}")
    return _DT_DENSE[dtype]


def _core_dtype(dtype: torch.dtype) -> torch.dtype:
    return torch.float32 if dtype in _DT_LOW else dtype


def _require_cuda(t: torch.Tensor, what: str):
    if not t.is_cuda:
        raise RuntimeError(f"{what}: tensor must live on a CUDA device (tntorch_b200 has no CPU path)")


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ws(nbytes: int, device) -> torch.Tensor:
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)


def _workspace(nbytes: int, device) -> torch.Tensor:
    """The workspace of a size a *_workspace_bytes query returned.  A size of 0 is the library refusing the call
    (NotImplementedError)."""
    if nbytes == 0:
        check(_lib.ERR_UNSUPPORTED)
    return _ws(nbytes, device)


def _ptr(t: Optional[torch.Tensor]) -> C.c_void_p:
    return C.c_void_p(0 if t is None else t.data_ptr())


def _rmax_list(rmax, nbonds: int) -> List[int]:
    """Reference convention (tensor.py:2027-2029): scalar or list of N-1; None = no cap."""
    if not hasattr(rmax, "__len__"):
        rmax = [rmax] * nbonds
    assert len(rmax) == nbonds
    out = []
    for r in rmax:
        if r is None:
            out.append(0)
        else:
            r = int(r)
            assert r >= 1
            out.append(min(r, 2**31 - 1))
    return out


def _tt_ranks(cores, what: str, boundary: bool = False, one_dtype: bool = True) -> List[int]:
    """The rank list [r_0, ..., r_N] of TT cores [r_k, I_k, r_{k+1}], the form the C-ABI takes them in.  The library
    reads core k as r_k x I_k x r_{k+1} from that list, so the cores must be CUDA tensors (RuntimeError), 3-D, on one
    device and, unless one_dtype=False, of one dtype, and their ranks must chain (ValueError).  With boundary=True,
    r_0 and r_N must be 1."""
    for c in cores:
        _require_cuda(c, what)
    if not cores or any(c.dim() != 3 for c in cores):
        raise ValueError(f"{what}: cores must be 3-D tensors [r, I, r']")
    c0 = cores[0]
    if any(c.device != c0.device for c in cores):
        raise ValueError(f"{what}: cores must share one CUDA device")
    if one_dtype and any(c.dtype != c0.dtype for c in cores):
        raise ValueError(f"{what}: cores must share one dtype")
    if any(cores[k].shape[2] != cores[k + 1].shape[0] for k in range(len(cores) - 1)):
        raise ValueError(f"{what}: core ranks do not match")
    ranks = [c0.shape[0]] + [c.shape[2] for c in cores]
    if boundary and (ranks[0] != 1 or ranks[-1] != 1):
        raise ValueError(f"{what}: boundary ranks must be 1, got {ranks[0]} and {ranks[-1]}")
    return ranks


def _slot_views(buf: torch.Tensor, offs, ranks, shape, base: int = 0) -> List[torch.Tensor]:
    """The cores a library call wrote into its slotted output `buf`: core k starts at offs[k] and is
    [ranks[base + k], shape[k], ranks[base + k + 1]] (base = i * (N + 1) for tensor i of a batch's rank list)."""
    out = []
    for k, n in enumerate(shape):
        r0, r1 = ranks[base + k], ranks[base + k + 1]
        out.append(buf[offs[k]: offs[k] + r0 * n * r1].view(r0, n, r1))
    return out


def _ttsvd_layout(shape: Sequence[int], rmax):
    """The dense TT-SVD's arguments and output layout for `shape` and `rmax`: the i64 shape, the i32 rank caps (a single
    0 for one mode), each core's offset in the cores buffer and that buffer's capacity in elements.  A shape the
    library cannot lay out raises ValueError."""
    N = len(shape)
    rm = _rmax_list(rmax, max(N - 1, 0))
    sh, rmc = i64(shape), i32(rm if N > 1 else [0])
    offs = (C.c_int64 * max(N, 1))()
    cap = lib().tnb_ttsvd_cores_capacity(N, sh, rmc, offs)
    if cap < 0:
        check(_lib.ERR_INVALID)
    return sh, rmc, offs, cap


def launch_count() -> int:
    return int(lib().tnb_launch_count())


def set_reserved_sms(n: int) -> None:
    """Leave n SMs free in the persistent kernels (useful with several decompositions in flight on different streams)."""
    lib().tnb_set_reserved_sms(int(n))


def measure_tf32_peak(reps: int = 200, per_commit: int = 64, trials: int = 5):
    """Dense TF32 mma.sync peak of the current GPU in TFLOP/s (csrc/peak_tf32.cuh)."""
    tf, ms = (C.c_double * 1)(), (C.c_double * 1)()
    check(lib().tnb_measure_tf32_peak(int(reps), int(per_commit), int(trials), tf, ms, _stream()))
    return float(tf[0]), float(ms[0])


def measure_wgmma_tf32_peak(reps: int = 64, per_commit: int = 64, trials: int = 5):
    """Dense TF32 wgmma (m64n256k8, A from registers) peak of the current GPU in TFLOP/s (csrc/peak_tf32.cuh)."""
    tf, ms = (C.c_double * 1)(), (C.c_double * 1)()
    check(lib().tnb_measure_wgmma_tf32_peak(int(reps), int(per_commit), int(trials), tf, ms, _stream()))
    return float(tf[0]), float(ms[0])


def measure_f64_mma_peak(reps: int = 200, per_commit: int = 64, trials: int = 5):
    """Dense fp64 mma.sync (m16n8k16 .f64, the MMA of tt_dot) peak of the current GPU in TFLOP/s (csrc/peak_tf32.cuh)."""
    tf, ms = (C.c_double * 1)(), (C.c_double * 1)()
    check(lib().tnb_measure_f64_mma_peak(int(reps), int(per_commit), int(trials), tf, ms, _stream()))
    return float(tf[0]), float(ms[0])


def has_tensorcore_path() -> bool:
    return bool(lib().tnb_has_tensorcore_path())


# --------------------------------------------------------------------------------------
def ttsvd(data: torch.Tensor, rmax=None, eps: float = 1e-14, batch_mode: bool = False, use_tensorcore: bool = True,
          return_info: bool = False, concurrent: bool = False, speculate: bool = True):
    """Dense tensor -> list of TT cores [r_{k-1}, I_k, r_k] (tn.Tensor(data, ranks_tt=...), tensor.py:401-408)."""
    _require_cuda(data, "ttsvd")
    data = data.contiguous()
    plan = TTSVDPlan(data.shape, data.dtype, rmax=rmax, device=data.device, use_tensorcore=use_tensorcore,
                     concurrent=concurrent, speculate=speculate, batch_mode=batch_mode)
    cores = plan.run(data, eps)
    if return_info:
        return cores, _ttsvd_info(plan.info)
    return cores


def _ttsvd_info(info) -> dict:
    return dict(norm=info[0], eig_solves=int(info[1]), chfsi_products=int(info[2]), tc_grams=int(info[3]),
                fused_filters=int(info[31]), rr_sweeps=int(info[29]), outer_iterations=int(info[30]),
                speculative=int(info[26]), spec_flags=int(info[27]), kblocked_steps=int(info[28]))


def ttsvd_stream(X_cpu: torch.Tensor, rmax=None, eps: float = 1e-14, chunk_bytes: Optional[int] = None,
                 return_info: bool = False):
    """Dense tensor in host memory -> TT cores on the current CUDA device, without ever holding the whole tensor there
    (tnb_ttsvd_stream): step 0 streams it through the device in chunks of about `chunk_bytes` (None: 256 MiB), the rest
    of the sweep runs as in `ttsvd`.  For tensors larger than free device memory.  `X_cpu`: a CPU tensor of any dtype
    `ttsvd` takes (pinned memory copies at full speed; pageable memory is staged through pinned pieces).  `info` is that
    of `ttsvd` plus `passes` (over the host tensor: 2, or 3 when the tensor-core step-0 Gram was rejected for the exact
    one) and `chunks` (per pass); its `norm` is ‖X‖_F, see `tt_relative_error_from_norm`."""
    if X_cpu.is_cuda:
        raise ValueError("ttsvd_stream: X_cpu must be a CPU tensor (decompose a device tensor with ttsvd)")
    X = X_cpu.contiguous()
    code = _dense_code(X.dtype)
    dev = torch.device("cuda", torch.cuda.current_device())
    N = X.dim()
    shape = list(X.shape)
    sh, rmc, offs, cap = _ttsvd_layout(shape, rmax)
    L = lib()
    cb = 0 if chunk_bytes is None else int(chunk_bytes)
    ws = _workspace(L.tnb_ttsvd_stream_workspace_bytes(code, N, sh, rmc, cb, 0), dev)
    cores_buf = torch.empty(int(cap), dtype=_core_dtype(X.dtype), device=dev)
    ranks = (C.c_int32 * (N + 1))()
    info = (C.c_double * 32)()
    with torch.cuda.device(dev):
        check(L.tnb_ttsvd_stream(code, _ptr(X), N, sh, rmc, float(eps), 0, cb, _ptr(ws), ws.numel(), _ptr(cores_buf), cap,
                                 ranks, info, _stream()))
    cores = _slot_views(cores_buf, offs, ranks, shape)
    if return_info:
        return cores, dict(_ttsvd_info(info), passes=int(info[24]), chunks=int(info[25]))
    return cores


def stream_instead_of_copy(input_bytes: int, workspace_bytes: int, free_bytes: int) -> bool:
    """The rule `tn.Tensor(X_cpu, ranks_tt=r)` decomposes by: stream the host tensor (`ttsvd_stream`) when its device
    image and the device call's workspace would not fit in free device memory, copy it and call `ttsvd` otherwise."""
    return input_bytes + workspace_bytes > free_bytes


def dot_instead_of_dense(dense_bytes: int, free_bytes: int) -> bool:
    """The rule `tn.relative_error(TT, TT)` measures by: the dot-product formula on the trains (tt_dot_batch) when the
    two dense tensors would not fit in free device memory, decompress both and compare them otherwise."""
    return dense_bytes > free_bytes


def tt_relative_error_from_norm(norm: float, cores: Sequence[torch.Tensor]) -> float:
    """‖T − TT(cores)‖_F / ‖T‖_F from ‖T‖_F alone (`info["norm"]` of `ttsvd` / `ttsvd_stream`), for cores in the TT-SVD
    gauge: cores 1…N−1 have orthonormal right unfoldings, so ‖T − T̂‖² = ‖T‖² − ‖core_0‖².  This is the error of a
    decomposition whose input never fits on the device.  It is only meaningful when the relative error is well above
    the resolution of ‖core_0‖² in the cores' precision: about 1e-3 for float32 cores (the difference of two squared
    norms loses the rest); below that, use `tt_relative_error` on the data."""
    norm = float(norm)
    if norm == 0.0:
        return 0.0
    c0 = float(torch.linalg.vector_norm(cores[0].detach().double()))
    return max(norm * norm - c0 * c0, 0.0) ** 0.5 / norm


class TTSVDPlan:
    """Pre-allocated buffers for repeated decompositions of one shape (bench.py, serving loops)."""

    def __init__(self, shape: Sequence[int], dtype: torch.dtype, rmax=None, device="cuda", use_tensorcore: bool = True,
                 host_io: bool = False, profile: bool = False, concurrent: bool = False, speculate: bool = True,
                 batch_mode: bool = False):
        self.shape = [int(s) for s in shape]
        self.N = len(self.shape)
        self.dtype = dtype
        self.device = torch.device(device)
        self.code = _dense_code(dtype)
        # concurrent: several plans run at once on different streams (TNB_FLAG_CONCURRENT, include/tnb200.h)
        self.flags = ((0 if use_tensorcore else _lib.FLAG_NO_TENSORCORE) | (_lib.FLAG_PROFILE if profile else 0) |
                      (_lib.FLAG_CONCURRENT if concurrent else 0) | (0 if speculate else _lib.FLAG_NO_SPECULATE) |
                      (_lib.FLAG_BATCH_MODE if batch_mode else 0))
        self._sh, self._rm, self._offs, self.cap = _ttsvd_layout(self.shape, rmax)
        self.ws = _workspace(lib().tnb_ttsvd_workspace_bytes(self.code, self.N, self._sh, self._rm, self.flags),
                             self.device)
        self.cores_buf = torch.empty(int(self.cap), dtype=_core_dtype(dtype), device=self.device)
        self.ranks = (C.c_int32 * (self.N + 1))()
        self.info = (C.c_double * 32)()
        self.numel = 1
        for s in self.shape:
            self.numel *= s
        self.dev_in = None
        self.cores_host = None
        if host_io:
            self.dev_in = torch.empty(self.numel, dtype=dtype, device=self.device)
            self.cores_host = torch.empty(int(self.cap), dtype=_core_dtype(dtype), pin_memory=True)

    def run(self, data: torch.Tensor, eps: float = 1e-14):
        with torch.cuda.device(self.device):
            check(lib().tnb_ttsvd(self.code, _ptr(data), self.N, self._sh, self._rm, float(eps), self.flags,
                                  _ptr(self.ws), self.ws.numel(), _ptr(self.cores_buf), self.cap, self.ranks, self.info,
                                  _stream()))
        return _slot_views(self.cores_buf, self._offs, self.ranks, self.shape)

    def run_host(self, data_host: torch.Tensor, eps: float = 1e-14):
        """End-to-end call on HOST buffers: H2D of the tensor, decomposition, D2H of the cores."""
        assert self.dev_in is not None, "construct the plan with host_io=True"
        with torch.cuda.device(self.device):
            check(lib().tnb_ttsvd_host(self.code, _ptr(data_host), self.N, self._sh, self._rm, float(eps), self.flags,
                                       _ptr(self.dev_in), _ptr(self.ws), self.ws.numel(), _ptr(self.cores_buf), self.cap,
                                       _ptr(self.cores_host), self.ranks, self.info, _stream()))
        return _slot_views(self.cores_host, self._offs, self.ranks, self.shape)


class TTSVDBatchPlan:
    """Pre-allocated buffers for decomposing batches of `batch` dense tensors of one shape through tnb_ttsvd_batch
    (tn.Tensor(X[B, ...], ranks_tt=r, batch=True); bench.py; dist.ttsvd_batch_sharded).  Up to `inflight` tensors are
    in flight at once inside the library (internal streams, one enqueueing thread, one synchronisation)."""

    def __init__(self, shape: Sequence[int], dtype: torch.dtype, batch: int, rmax=None, device="cuda", inflight: int = 8,
                 use_tensorcore: bool = True, batch_mode: bool = False, host_io: bool = False):
        self.shape = [int(s) for s in shape]
        self.N = len(self.shape)
        self.batch = int(batch)
        self.dtype = dtype
        self.device = torch.device(device)
        self.code = _dense_code(dtype)
        self.flags = (0 if use_tensorcore else _lib.FLAG_NO_TENSORCORE) | (_lib.FLAG_BATCH_MODE if batch_mode else 0)
        self._sh, self._rm, self._offs, self.cap = _ttsvd_layout(self.shape, rmax)
        one = C.c_size_t(0)
        lib().tnb_ttsvd_batch_workspace_bytes(self.code, self.batch, self.N, self._sh, self._rm, self.flags, C.byref(one))
        self.per_tensor_bytes = int(one.value)
        self.inflight = max(1, min(int(inflight), self.batch, 8))
        self.ws = _workspace(self.per_tensor_bytes * self.inflight, self.device)
        self.cores_buf = torch.empty(self.batch, int(self.cap), dtype=_core_dtype(dtype), device=self.device)
        self.ranks = (C.c_int32 * (self.batch * (self.N + 1)))()
        self.norms = (C.c_double * self.batch)()
        self.spec = (C.c_int32 * self.batch)()
        self.numel = 1
        for s in self.shape:
            self.numel *= s
        self._cores_ptrs = (C.c_void_p * self.batch)(*[self.cores_buf[i].data_ptr() for i in range(self.batch)])
        self.dev_in = None
        self.cores_host = None
        if host_io:
            self.dev_in = torch.empty(self.batch, self.numel, dtype=dtype, device=self.device)
            self.cores_host = torch.empty(self.batch, int(self.cap), dtype=_core_dtype(dtype), pin_memory=True)

    def run(self, tensors, eps: float = 1e-14):
        """tensors: a [batch, ...] tensor or a sequence of `batch` contiguous device tensors.  Returns, per tensor, the
        list of its cores (views of the plan's buffers: valid until the next run)."""
        if isinstance(tensors, torch.Tensor):
            tensors = [tensors[i] for i in range(tensors.shape[0])]
        assert len(tensors) == self.batch
        keep = [t if t.is_contiguous() else t.contiguous() for t in tensors]
        ptrs = (C.c_void_p * self.batch)(*[t.data_ptr() for t in keep])
        with torch.cuda.device(self.device):
            check(lib().tnb_ttsvd_batch(self.code, ptrs, self.batch, self.N, self._sh, self._rm, float(eps), self.flags,
                                        _ptr(self.ws), self.ws.numel(), self._cores_ptrs, self.cap, self.ranks, self.norms,
                                        self.spec, _stream()))
        return [_slot_views(self.cores_buf[i], self._offs, self.ranks, self.shape, i * (self.N + 1))
                for i in range(self.batch)]

    def run_host(self, tensors_host: torch.Tensor, eps: float = 1e-14):
        """End to end on HOST buffers: `tensors_host` [batch, ...] in (pinned) host memory -> device, decomposition,
        cores back to pinned host memory.  The copy of tensor i+1 overlaps nothing here (one stream): the PCIe link is
        the bound either way."""
        assert self.dev_in is not None, "construct the plan with host_io=True"
        flat = tensors_host.reshape(self.batch, self.numel)
        self.dev_in.copy_(flat, non_blocking=True)
        self.run(self.dev_in.view([self.batch] + self.shape), eps)
        self.cores_host.copy_(self.cores_buf, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return [_slot_views(self.cores_host[i], self._offs, self.ranks, self.shape, i * (self.N + 1))
                for i in range(self.batch)]


def ttsvd_batch(tensors, rmax=None, eps: float = 1e-14, batch_mode: bool = False, inflight: int = 8,
                use_tensorcore: bool = True, return_info: bool = False):
    """Decompose a batch of dense tensors of one shape (a [B, ...] tensor or a sequence): tn.Tensor(..., batch=True)
    and every caller that decomposes many tensors.  Returns a list (per tensor) of lists of cores (fresh tensors)."""
    if isinstance(tensors, torch.Tensor):
        tensors = [tensors[i] for i in range(tensors.shape[0])]
    if len(tensors) == 0:
        return ([], dict(speculative=[])) if return_info else []
    t0 = tensors[0]
    _require_cuda(t0, "ttsvd_batch")
    for t in tensors:
        if t.shape != t0.shape or t.dtype != t0.dtype or t.device != t0.device:
            raise ValueError("ttsvd_batch: all tensors must share shape, dtype and device")
    plan = TTSVDBatchPlan(t0.shape, t0.dtype, len(tensors), rmax=rmax, device=t0.device, inflight=inflight,
                          use_tensorcore=use_tensorcore, batch_mode=batch_mode)
    views = plan.run(tensors, eps)
    out = [[c.clone() for c in cores] for cores in views]
    if return_info:
        return out, dict(speculative=[int(x) for x in plan.spec], norms=[float(x) for x in plan.norms])
    return out


# --------------------------------------------------------------------------------------
def tt_round(cores: Sequence[torch.Tensor], eps: float = 1e-14, rmax=None, batch_mode: bool = False,
             speculate: bool = True):
    """Tensor.round_tt on device cores (tensor.py:2008-2083). Returns new cores.  speculate=False runs the host-driven
    sweeps even where the speculative one-synchronisation path is eligible (TNB_FLAG_NO_SPECULATE)."""
    N = len(cores)
    rin = _tt_ranks(cores, "tt_round")
    dt = cores[0].dtype
    cores = [c.contiguous() for c in cores]
    code = _dtype_code(cores[0])
    shape = [c.shape[1] for c in cores]
    rm = _rmax_list(rmax, max(N - 1, 0))
    L = lib()
    sh, rinc = i64(shape), i32(rin)
    rmc = i32(rm) if N > 1 else i32([0])
    offs = (C.c_int64 * N)()
    cap = L.tnb_tt_round_cores_capacity(N, sh, rinc, rmc, offs)
    if cap < 0:
        check(_lib.ERR_INVALID)
    dev = cores[0].device
    ws = _workspace(L.tnb_tt_round_workspace_bytes(code, N, sh, rinc, rmc), dev)
    out = torch.empty(int(cap), dtype=dt, device=dev)
    ranks = (C.c_int32 * (N + 1))()
    ptrs = (C.c_void_p * N)(*[c.data_ptr() for c in cores])
    flags = (_lib.FLAG_BATCH_MODE if batch_mode else 0) | (0 if speculate else _lib.FLAG_NO_SPECULATE)
    with torch.cuda.device(dev):
        check(L.tnb_tt_round(code, ptrs, N, sh, rinc, rmc, float(eps), flags, _ptr(ws), ws.numel(), _ptr(out), cap, ranks,
                             _stream()))
    return _slot_views(out, offs, ranks, shape)


def tt_round_batch(batch_cores: Sequence[Sequence[torch.Tensor]], eps: float = 1e-14, rmax=None, batch_mode: bool = False,
                   inflight: int = 8, return_info: bool = False, speculate: bool = True):
    """Round a batch of TT tensors that share shape and input ranks: ONE library call, several tensors in flight
    (tnb_tt_round_batch).  batch_cores: per tensor, its list of cores [r, I, r'].  Returns per tensor the new cores.

    return_info adds dict(speculative=[...]): 1 where a tensor's result came from the speculative sweeps (one
    synchronisation), 0 where it came from the host-driven sweeps.  With one tensor the call goes through the same
    dispatcher as tt_round, so this reports which path tt_round takes on that input; with B > 1 and inflight >= 2 it
    goes through the in-flight driver, which redoes each tensor whose speculation failed on the host-driven path.
    speculate=False runs the host-driven sweeps for every tensor (TNB_FLAG_NO_SPECULATE)."""
    B = len(batch_cores)
    if B == 0:
        return []
    N = len(batch_cores[0])
    cs = [[c.contiguous() for c in cores] for cores in batch_cores]
    for cores in cs:
        rin = _tt_ranks(cores, "tt_round_batch")
        if ([c.shape for c in cores] != [c.shape for c in cs[0]] or cores[0].dtype != cs[0][0].dtype
                or cores[0].device != cs[0][0].device):
            raise ValueError("tt_round_batch: all tensors must share their core shapes, dtype and device")
    dt, dev = cs[0][0].dtype, cs[0][0].device
    code = _dtype_code(cs[0][0])
    shape = [c.shape[1] for c in cs[0]]
    rm = _rmax_list(rmax, max(N - 1, 0))
    L = lib()
    sh, rinc = i64(shape), i32(rin)
    rmc = i32(rm) if N > 1 else i32([0])
    offs = (C.c_int64 * N)()
    cap = L.tnb_tt_round_cores_capacity(N, sh, rinc, rmc, offs)
    if cap < 0:
        check(_lib.ERR_INVALID)
    one = C.c_size_t(0)
    L.tnb_tt_round_batch_workspace_bytes(code, B, N, sh, rinc, rmc, C.byref(one))
    k = max(1, min(int(inflight), B, 8))
    ws = _workspace(one.value * k, dev)
    out = torch.empty(B, int(cap), dtype=dt, device=dev)
    ranks = (C.c_int32 * (B * (N + 1)))()
    spec = (C.c_int32 * B)()
    pin = (C.c_void_p * (B * N))(*[c.data_ptr() for cores in cs for c in cores])
    pout = (C.c_void_p * B)(*[out[i].data_ptr() for i in range(B)])
    flags = (_lib.FLAG_BATCH_MODE if batch_mode else 0) | (0 if speculate else _lib.FLAG_NO_SPECULATE)
    with torch.cuda.device(dev):
        check(L.tnb_tt_round_batch(code, pin, B, N, sh, rinc, rmc, float(eps), flags, _ptr(ws), ws.numel(), pout, cap, ranks, spec,
                                   _stream()))
    res = [_slot_views(out[i], offs, ranks, shape, i * (N + 1)) for i in range(B)]
    if return_info:
        return res, dict(speculative=[int(x) for x in spec])
    return res


def _tt_operands(operands, what: str, boundary: bool = False):
    """operands: list of lists of TT cores [r, I, r'] (same shape, dtype, device) -> pointers / ranks for the C-ABI."""
    K = len(operands)
    N = len(operands[0])
    ops_c = [[c.contiguous() for c in cores] for cores in operands]
    ranks = []
    for cores in ops_c:
        ranks += _tt_ranks(cores, what, boundary)
    dt, dev = ops_c[0][0].dtype, ops_c[0][0].device
    shape = [c.shape[1] for c in ops_c[0]]
    for cores in ops_c:
        if len(cores) != N or [c.shape[1] for c in cores] != shape:
            raise ValueError("TT operands must share their shape")
        if cores[0].dtype != dt or cores[0].device != dev:
            raise ValueError("TT operands must be lists of [r, I, r'] cores of one dtype on one device")
    ptrs = (C.c_void_p * (K * N))(*[c.data_ptr() for cores in ops_c for c in cores])
    return ops_c, K, N, shape, ranks, ptrs, dt, dev


def tt_sum(operands, alpha=None):
    """sum_k alpha_k T_k as block TT cores (Tensor.__add__, tensor.py:445-520); no rounding."""
    ops_c, K, N, shape, ranks, ptrs, dt, dev = _tt_operands(operands, "tt_sum")
    L = lib()
    rsum = (C.c_int32 * (N + 1))()
    offs = (C.c_int64 * N)()
    cap = L.tnb_tt_sum_cores_capacity(K, N, i64(shape), i32(ranks), rsum, offs)
    if cap < 0:
        check(_lib.ERR_INVALID)
    out = torch.empty(int(cap), dtype=dt, device=dev)
    al = None if alpha is None else (C.c_double * K)(*[float(a) for a in alpha])
    with torch.cuda.device(dev):
        check(L.tnb_tt_sum(_dtype_code(ops_c[0][0]), ptrs, K, al, N, i64(shape), i32(ranks), _ptr(out), cap, _stream()))
    return _slot_views(out, offs, rsum, shape)


def tt_sum_round(operands, alpha=None, eps: float = 1e-14, rmax=None, speculate: bool = True):
    """round_tt(sum_k alpha_k T_k) in ONE library call: block cores assembled in the workspace, then the rounding sweeps
    (the `tn.round(function(a, b))` step of tools.reduce, tools.py:460-512).  speculate as for tt_round."""
    ops_c, K, N, shape, ranks, ptrs, dt, dev = _tt_operands(operands, "tt_sum_round")
    L = lib()
    rm = _rmax_list(rmax, max(N - 1, 0))
    rmc = i32(rm) if N > 1 else i32([0])
    offs = (C.c_int64 * N)()
    cap = L.tnb_tt_sum_round_cores_capacity(K, N, i64(shape), i32(ranks), rmc, offs)
    if cap < 0:
        check(_lib.ERR_INVALID)
    code = _dtype_code(ops_c[0][0])
    ws = _workspace(L.tnb_tt_sum_round_workspace_bytes(code, K, N, i64(shape), i32(ranks), rmc), dev)
    out = torch.empty(int(cap), dtype=dt, device=dev)
    rk = (C.c_int32 * (N + 1))()
    al = None if alpha is None else (C.c_double * K)(*[float(a) for a in alpha])
    flags = 0 if speculate else _lib.FLAG_NO_SPECULATE
    with torch.cuda.device(dev):
        check(L.tnb_tt_sum_round(code, ptrs, K, al, N, i64(shape), i32(ranks), rmc, float(eps), flags, _ptr(ws), ws.numel(), _ptr(out),
                                 cap, rk, _stream()))
    return _slot_views(out, offs, rk, shape)


def tt_hadamard(a_cores, b_cores):
    """Elementwise product of two TT tensors: Kronecker cores (Tensor.__mul__, tensor.py:560-640)."""
    ops_c, K, N, shape, ranks, ptrs, dt, dev = _tt_operands([a_cores, b_cores], "tt_hadamard")
    ra, rb = ranks[: N + 1], ranks[N + 1:]
    outs = [torch.empty(ra[n] * rb[n], shape[n], ra[n + 1] * rb[n + 1], dtype=dt, device=dev) for n in range(N)]
    pa = (C.c_void_p * N)(*[c.data_ptr() for c in ops_c[0]])
    pb = (C.c_void_p * N)(*[c.data_ptr() for c in ops_c[1]])
    po = (C.c_void_p * N)(*[c.data_ptr() for c in outs])
    with torch.cuda.device(dev):
        check(lib().tnb_tt_hadamard(_dtype_code(ops_c[0][0]), pa, pb, N, i64(shape), i32(ra), i32(rb), po, _stream()))
    return outs


def tt_hadamard_round(a_cores, b_cores, eps: float = 1e-14, rmax=None, return_info: bool = False,
                      use_tensorcore: bool = True):
    """round_tt(a * b) of two tensor trains in ONE library call (tnb_tt_hadamard_round) that never forms the Kronecker
    cores of the product: left Grams of the product by a structured recurrence, then the truncation sweep of tt_round on
    the Gram of each bond's carry.  Ranks and tolerance follow tt_round (delta = eps / sqrt(N - 1) ||a * b||, rmax a
    scalar or N - 1 caps).  fp32 or fp64 cores of one dtype (ValueError otherwise), computed in fp64, returned in the
    input dtype.  return_info adds dict(norm_sq=||a*b||^2, discarded_sq=||a*b - result||^2).  Envelope: a bond Gram of
    I_mu r_{mu+1} up to 46000 and, where it is wider than 256, a kept rank up to 240 (NotImplementedError otherwise):
    eps-only calls at large ranks need rmax.  use_tensorcore=False runs every GEMM on CUDA-core tiles."""
    ops_c, K, N, shape, ranks, ptrs, dt, dev = _tt_operands([a_cores, b_cores], "tt_hadamard_round", boundary=True)
    ra, rb = ranks[: N + 1], ranks[N + 1:]
    if any(c.requires_grad for cores in ops_c for c in cores):
        raise ValueError("tt_hadamard_round: cores that require grad are not supported")
    code = _dtype_code(ops_c[0][0])
    rm = _rmax_list(rmax, max(N - 1, 0))
    L = lib()
    sh, rac, rbc = i64(shape), i32(ra), i32(rb)
    rmc = i32(rm) if N > 1 else i32([0])
    offs = (C.c_int64 * N)()
    cap = L.tnb_tt_hadamard_round_cores_capacity(N, sh, rac, rbc, rmc, offs)
    if cap < 0:
        check(_lib.ERR_INVALID)
    ws = _workspace(L.tnb_tt_hadamard_round_workspace_bytes(code, N, sh, rac, rbc, rmc), dev)
    out = torch.empty(int(cap), dtype=dt, device=dev)
    rk = (C.c_int32 * (N + 1))()
    en = (C.c_double * 2)()
    pa = (C.c_void_p * N)(*[c.data_ptr() for c in ops_c[0]])
    pb = (C.c_void_p * N)(*[c.data_ptr() for c in ops_c[1]])
    flags = 0 if use_tensorcore else _lib.FLAG_NO_TENSORCORE
    with torch.cuda.device(dev):
        check(L.tnb_tt_hadamard_round(code, pa, pb, N, sh, rac, rbc, rmc, float(eps), flags, _ptr(ws), ws.numel(), _ptr(out),
                                      cap, rk, en, _stream()))
    res = _slot_views(out, offs, rk, shape)
    if return_info:
        return res, dict(norm_sq=float(en[0]), discarded_sq=float(en[1]))
    return res


def hadamard_round_instead_of_kronecker(shape: Sequence[int], ranks_a: Sequence[int], ranks_b: Sequence[int],
                                        itemsize: int, free_bytes: int) -> bool:
    """The rule `round_tt(a * b)` inside `tn.reduce(..., operator.mul)` and `tn.hadamard_sum(..., 'svd' | 'eig')` is
    computed by: the fused `tt_hadamard_round` when the Kronecker path cannot run, i.e. some product rank
    ra_k rb_k is above 256 (tt_round's direct eigensolver limit), or the Kronecker cores plus tt_round's workspace
    exceed free device memory; the Kronecker cores (`tt_hadamard`) and `tt_round` otherwise."""
    N = len(shape)
    R = [int(a) * int(b) for a, b in zip(ranks_a, ranks_b)]
    if any(r > 256 for r in R):
        return True
    kron = sum(R[k] * int(shape[k]) * R[k + 1] for k in range(N)) * int(itemsize)
    code = _lib.TNB_F32 if int(itemsize) == 4 else _lib.TNB_F64
    rm = i32([0] * max(N - 1, 1))
    wsb = lib().tnb_tt_round_workspace_bytes(code, N, i64(shape), i32(R), rm)
    if wsb == 0:
        return True
    cap = lib().tnb_tt_round_cores_capacity(N, i64(shape), i32(R), rm, None)
    return kron + int(wsb) + max(int(cap), 0) * int(itemsize) > int(free_bytes)


def truncated_svd(M: torch.Tensor, delta=None, eps=None, rmax=None, left_ortho=True, batch_mode: bool = False,
                  return_zero_flag: bool = False):
    """tn.truncated_svd (round.py:52-187) of one matrix.  batch_mode = the reference's rank rule for one sample of a
    batch (round.py:149-150); return_zero_flag additionally returns whether the sample was numerically zero."""
    if delta is not None and eps is not None:
        raise ValueError("Provide either `delta` or `eps`")
    _require_cuda(M, "truncated_svd")
    if M.dim() != 2:
        raise ValueError("truncated_svd expects a matrix")
    M = M.contiguous()
    code = _dtype_code(M)
    m, n = M.shape
    if rmax is None:
        rm = 0
    else:
        assert rmax >= 1
        rm = int(min(rmax, 2**31 - 1))
    L = lib()
    ws = _workspace(L.tnb_truncated_svd_workspace_bytes(code, m, n), M.device)
    k = min(m, n)
    left = torch.empty(m * k, dtype=M.dtype, device=M.device)
    right = torch.empty(k * n, dtype=M.dtype, device=M.device)
    rank = (C.c_int32 * 1)()
    with torch.cuda.device(M.device):
        check(L.tnb_truncated_svd(code, _ptr(M), m, n, -1.0 if delta is None else float(delta),
                                  -1.0 if eps is None else float(eps), rm, (1 if left_ortho else 0) | (2 if batch_mode else 0),
                                  _ptr(ws), ws.numel(), _ptr(left), _ptr(right), rank, _stream()))
    r = abs(rank[0])
    out = left[: m * r].view(m, r), right[: r * n].view(r, n)
    return out + (rank[0] < 0,) if return_zero_flag else out


def cp_als(data: torch.Tensor, R: int, max_iter: int = 25, tol: float = 1e-4, return_info: bool = False, init=None):
    """CP-ALS on the device (tn.Tensor(data, ranks_cp=R, max_iter=, tol=), tensor.py:210-400).
    Returns the list of factor matrices [I_n, R].  init: optional list of starting factors [I_n, R] (CP on a Tucker
    core starts from random factors, tensor.py:278-302); default: the HOSVD initialisation of tensor.py:217-277."""
    _require_cuda(data, "cp_als")
    data = data.contiguous()
    code = _dtype_code(data)
    N = data.dim()
    shape = list(data.shape)
    L = lib()
    sh = i64(shape)
    offs = (C.c_int64 * N)()
    cap = L.tnb_cp_als_factors_capacity(N, sh, int(R), offs)
    if cap < 0:
        check(_lib.ERR_INVALID if N >= 2 else _lib.ERR_UNSUPPORTED)
    ws = _workspace(L.tnb_cp_als_workspace_bytes(code, N, sh, int(R)), data.device)
    fac = torch.zeros(int(cap), dtype=data.dtype, device=data.device)
    errs = (C.c_double * max(int(max_iter), 1))()
    iters = (C.c_int32 * 1)()
    entry = L.tnb_cp_als
    if init is not None:
        assert len(init) == N
        for n in range(N):
            assert tuple(init[n].shape) == (shape[n], int(R))
            fac[offs[n]: offs[n] + shape[n] * R].copy_(init[n].to(device=data.device, dtype=data.dtype).reshape(-1))
        entry = L.tnb_cp_als_from
    with torch.cuda.device(data.device):
        check(entry(code, _ptr(data), N, sh, int(R), int(max_iter), float(tol), _ptr(ws), ws.numel(), _ptr(fac), cap,
                    errs, iters, _stream()))
    factors = [fac[offs[n]: offs[n] + shape[n] * R].view(shape[n], R) for n in range(N)]
    if return_info:
        return factors, dict(errors=[errs[i] for i in range(iters[0])], iters=int(iters[0]))
    return factors


def maxvol(A: torch.Tensor, tol: float = 1.05, max_iters: int = 100, return_iters: bool = False):
    """Device maxvol (tntorch/maxvol.py:114-170).  A: [N, r] or a batch [B, N, r].  Returns (index int32 [.., min(N,r)],
    C [.., N, r] = A inv(A[index])) as device tensors; nothing is copied to the host."""
    _require_cuda(A, "maxvol")
    batched = A.dim() == 3
    A3 = (A if batched else A[None]).contiguous().double()
    B, N, r = A3.shape
    L = lib()
    ws = _ws(L.tnb_maxvol_workspace_bytes(B, N, r), A.device)
    index = torch.empty(B, r, dtype=torch.int32, device=A.device)
    Cm = torch.empty(B, N, r, dtype=torch.float64, device=A.device)
    iters = (C.c_int32 * B)() if return_iters else None
    with torch.cuda.device(A.device):
        check(L.tnb_maxvol(_ptr(A3), B, N, r, float(tol), int(max_iters), _ptr(ws), ws.numel(), _ptr(index), _ptr(Cm), iters,
                           _stream()))
    if N <= r:  # maxvol.py:126-127
        index, Cm = index[:, :N], Cm[:, :, :N]
    if not batched:
        index, Cm = index[0], Cm[0]
    if return_iters:
        return index, Cm, [int(x) for x in iters]
    return index, Cm


def rect_maxvol(A: torch.Tensor, tol: float = 1.0, maxK=None, min_add_K=None, minK=None, start_maxvol_iters: int = 10):
    """Device rect_maxvol (tntorch/maxvol.py:30-111).  A: [N, r] or a batch [B, N, r].  Returns (index, C) like the
    reference: the chosen rows (int32) and the coefficient matrix [N, K] with identity rows at the chosen positions; for
    a batch, lists of per-problem results (K is data dependent)."""
    _require_cuda(A, "rect_maxvol")
    batched = A.dim() == 3
    A3 = (A if batched else A[None]).contiguous().double()
    B, N, r = A3.shape
    if N <= r:  # maxvol.py:52-53
        out = [(torch.arange(N, dtype=torch.int32, device=A.device), torch.eye(N, dtype=torch.float64, device=A.device))
               for _ in range(B)]
        return out if batched else out[0]
    # parameter normalisation of maxvol.py:54-66
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
    L = lib()
    ws = _ws(L.tnb_rect_maxvol_workspace_bytes(B, N, r, int(maxK)), A.device)
    index = torch.empty(B, int(maxK), dtype=torch.int32, device=A.device)
    Cm = torch.empty(B, N, int(maxK), dtype=torch.float64, device=A.device)
    Kd = torch.empty(B, dtype=torch.int32, device=A.device)
    with torch.cuda.device(A.device):
        check(L.tnb_rect_maxvol(_ptr(A3), B, N, r, float(tol), int(minK), int(maxK), int(start_maxvol_iters), _ptr(ws),
                                ws.numel(), _ptr(index), _ptr(Cm), _ptr(Kd), _stream()))
    Ks = Kd.tolist()
    out = [(index[b, : Ks[b]], Cm[b, :, : Ks[b]]) for b in range(B)]
    return out if batched else out[0]


# ---- batched TT-cross plumbing (cross_batch.py) -----------------------------------------------------------------------
def cross_gather_coords(lsets: torch.Tensor, rsets: torch.Tensor, grid: torch.Tensor, N: int, j: int, I: int):
    """lsets [B, Rl, j] / rsets [B, Rr, N-j-1] int32, grid [N, Imax] fp64 -> N coordinate vectors of length B*Rl*I*Rr."""
    B, Rl, Rr = lsets.shape[0], lsets.shape[1], rsets.shape[1]
    X = torch.empty(N, B * Rl * I * Rr, dtype=torch.float64, device=grid.device)
    lsets, rsets = lsets.contiguous(), rsets.contiguous()
    with torch.cuda.device(grid.device):
        check(lib().tnb_cross_gather_coords(_ptr(lsets), _ptr(rsets), _ptr(grid), grid.shape[1], B, N, j, Rl, I, Rr, _ptr(X),
                                            _stream()))
    return [X[k] for k in range(N)]


def cross_update_lsets(lsets: torch.Tensor, local: torch.Tensor, I: int, active=None, old=None):
    B, Rl, j = lsets.shape
    Rn = local.shape[1]
    out = old if (old is not None and active is not None) else torch.empty(B, Rn, j + 1, dtype=torch.int32, device=local.device)
    lsets, local = lsets.contiguous(), local.contiguous()
    with torch.cuda.device(local.device):
        check(lib().tnb_cross_update_lsets(_ptr(lsets), _ptr(local), B, j, Rl, I, Rn, _ptr(active) if old is not None else _ptr(None),
                                           _ptr(out), _stream()))
    return out


def cross_update_rsets(rsets: torch.Tensor, local: torch.Tensor, Rr: int, active=None, old=None):
    B, _, ln = rsets.shape  # suffix of modes j+1..N-1
    Rp = local.shape[1]
    out = old if (old is not None and active is not None) else torch.empty(B, Rp, ln + 1, dtype=torch.int32, device=local.device)
    rsets, local = rsets.contiguous(), local.contiguous()
    # N and j only enter through N - j - 1 = ln: pass (N, j) = (ln + 2, 1)
    I = 0
    with torch.cuda.device(local.device):
        check(lib().tnb_cross_update_rsets(_ptr(rsets), _ptr(local), B, ln + 2, 1, 1 << 30, Rr, Rp,
                                           _ptr(active) if old is not None else _ptr(None), _ptr(out), _stream()))
    return out


def cross_tt_eval(cores: Sequence[torch.Tensor], idx: torch.Tensor) -> torch.Tensor:
    """cores: N tensors [B, r, I, r'] fp64; idx: [P, N] (shared) or [B, P, N] int32 -> values [B, P]."""
    N = len(cores)
    B = cores[0].shape[0]
    per = idx.dim() == 3
    P = idx.shape[-2]
    cs = [c.contiguous() for c in cores]
    idx = idx.contiguous()
    out = torch.empty(B, P, dtype=torch.float64, device=cs[0].device)
    ptrs = (C.c_void_p * N)(*[c.data_ptr() for c in cs])
    ranks = i32([cs[0].shape[1]] + [c.shape[3] for c in cs])
    shape = i32([c.shape[2] for c in cs])
    with torch.cuda.device(cs[0].device):
        check(lib().tnb_cross_tt_eval(ptrs, N, ranks, shape, _ptr(idx), B, P, 1 if per else 0, _ptr(out), _stream()))
    return out


def matmul(A: torch.Tensor, B: torch.Tensor) -> torch.Tensor:
    """Row-major A @ B on the library's own GEMM (no cuBLAS)."""
    _require_cuda(A, "matmul")
    A, B = A.contiguous(), B.contiguous()
    assert A.dtype == B.dtype and A.shape[1] == B.shape[0]
    M, K = A.shape
    N = B.shape[1]
    Cm = torch.empty(M, N, dtype=A.dtype, device=A.device)
    with torch.cuda.device(A.device):
        check(lib().tnb_matmul(_dtype_code(A), _ptr(A), _ptr(B), _ptr(Cm), M, N, K, _stream()))
    return Cm


def qr(A: torch.Tensor, return_r: bool = False):
    """Householder QR on the device (torch.linalg.qr semantics, reduced): A [rows, n] or batch [B, rows, n], fp64."""
    _require_cuda(A, "qr")
    batched = A.dim() == 3
    A3 = (A if batched else A[None]).contiguous().double()
    B, rows, n = A3.shape
    k = min(rows, n)
    L = lib()
    ws = _ws(L.tnb_qr_workspace_bytes(B, rows, n), A.device)
    Q = torch.empty(B, rows, k, dtype=torch.float64, device=A.device)
    R = torch.empty(B, k, n, dtype=torch.float64, device=A.device) if return_r else None
    with torch.cuda.device(A.device):
        check(L.tnb_qr_householder(_ptr(A3), B, rows, n, _ptr(ws), ws.numel(), _ptr(Q), _ptr(R), _stream()))
    if not batched:
        Q = Q[0]
        R = R[0] if return_r else None
    return (Q, R) if return_r else Q


def gram(A: torch.Tensor, tensorcore: bool = False) -> torch.Tensor:
    """fp64 Gram matrix A^T A of a (rows x n) matrix; tensorcore=True uses the TMA tensor-core kernel (fp32 only)."""
    _require_cuda(A, "gram")
    A = A.contiguous()
    rows, n = A.shape
    G = torch.empty(n, n, dtype=torch.float64, device=A.device)
    L = lib()
    with torch.cuda.device(A.device):
        if tensorcore:
            if A.dtype != torch.float32:
                raise ValueError("tensor-core Gram needs float32 input")
            ws = _workspace(L.tnb_gram_tc_workspace_bytes(rows, n), A.device)
            check(L.tnb_gram_tc_f32(_ptr(A), rows, n, _ptr(G), _ptr(ws), ws.numel(), _stream()))
        else:
            code = _dtype_code(A)
            ws = _ws(L.tnb_gram_workspace_bytes(code, rows, n), A.device)
            check(L.tnb_gram(code, _ptr(A), rows, n, _ptr(G), _ptr(ws), ws.numel(), _stream()))
    return G


def to_kblocked(M: torch.Tensor) -> torch.Tensor:
    """The K-blocked storage of a (rows x n) matrix (rows, n multiples of 8): wgmma's K-major 8 x 4 core matrices,
    [rows/8][n/8][2][8][4], element (k, c) at (((k/8 * n/8 + c/8) * 2 + k%8/4) * 8 + c%8) * 4 + k%4."""
    rows, n = M.shape
    return M.reshape(rows // 8, 2, 4, n // 8, 8).permute(0, 3, 1, 4, 2).contiguous()


def from_kblocked(B: torch.Tensor, rows: int, n: int) -> torch.Tensor:
    """The (rows x n) matrix stored K-blocked in B (inverse of to_kblocked)."""
    return B.reshape(rows // 8, n // 8, 2, 8, 4).permute(0, 2, 4, 1, 3).reshape(rows, n)


def gram_kblocked(B: torch.Tensor, rows: int, n: int) -> torch.Tensor:
    """fp64 A^T A of the (rows x n) fp32 matrix A stored K-blocked in B (to_kblocked), on the tensor-core Gram kernel
    that reads both operands K-major (n >= 256, rows % 8 == 0)."""
    _require_cuda(B, "gram_kblocked")
    assert B.dtype == torch.float32 and B.is_contiguous() and B.numel() == rows * n
    G = torch.empty(n, n, dtype=torch.float64, device=B.device)
    L = lib()
    ws = _workspace(L.tnb_gram_tc_workspace_bytes(rows, n), B.device)
    with torch.cuda.device(B.device):
        check(L.tnb_gram_tc_kblocked_f32(_ptr(B), rows, n, _ptr(G), _ptr(ws), ws.numel(), _stream()))
    return G


# The 16- and 8-bit tensor-core Gram and projection of each input dtype: (Gram sizing query, Gram entry point,
# projection entry point, leading arguments).  Both float8 formats share entry points that take the format's code.
_TC_LOWP = {
    torch.bfloat16: ("tnb_gram_tc_bf16_workspace_bytes", "tnb_gram_tc_bf16", "tnb_project_tc_bf16", ()),
    torch.float16: ("tnb_gram_tc_f16_workspace_bytes", "tnb_gram_tc_f16", "tnb_project_tc_f16", ()),
    **{dt: ("tnb_gram_tc_f8_workspace_bytes", "tnb_gram_tc_f8", "tnb_project_tc_f8", (code,))
       for dt, code in _DT_F8.items()},
}


def _gram_lowp(A: torch.Tensor) -> torch.Tensor:
    """gram_bf16 / gram_f16 / gram_f8 on a CUDA matrix of their dtype."""
    size, gram, _, lead = _TC_LOWP[A.dtype]
    A = A.contiguous()
    rows, n = A.shape
    G = torch.empty(n, n, dtype=torch.float64, device=A.device)
    L = lib()
    ws = _workspace(getattr(L, size)(rows, n), A.device)
    with torch.cuda.device(A.device):
        check(getattr(L, gram)(*lead, _ptr(A), rows, n, _ptr(G), _ptr(ws), ws.numel(), _stream()))
    return G


def gram_bf16(A: torch.Tensor) -> torch.Tensor:
    """fp64 A^T A of a row-major bfloat16 (rows x n) matrix on the bf16 tensor-core Gram kernel (exact products, fp32
    accumulation): n % 8 == 0 and n = 32 / 64 (rows divisible by 128 / n), 128 or >= 256."""
    _require_cuda(A, "gram_bf16")
    assert A.dtype == torch.bfloat16
    return _gram_lowp(A)


def gram_f16(A: torch.Tensor) -> torch.Tensor:
    """fp64 A^T A of a row-major float16 (rows x n) matrix on the tensor-core Gram kernel with fp16 operands (exact
    products, fp32 accumulation); the shapes of gram_bf16."""
    _require_cuda(A, "gram_f16")
    assert A.dtype == torch.float16
    return _gram_lowp(A)


def gram_f8(A: torch.Tensor) -> torch.Tensor:
    """fp64 A^T A of a row-major float8 (e4m3fn or e5m2, rows x n) matrix on the tensor-core Gram kernel, the values
    widened to fp16 in shared memory (exact products, fp32 accumulation); the shapes of gram_bf16 with n % 16 == 0."""
    _require_cuda(A, "gram_f8")
    assert A.dtype in _DT_F8
    return _gram_lowp(A)


def gram_noise_level(dtype: torch.dtype) -> float:
    """||G_tc - (1 - c) G|| / ||G|| the TT-SVD's accept rule allows for the tensor-core Gram of float32 (TF32),
    bfloat16, float16 or float8 (e4m3fn, e5m2) input."""
    return float(lib().tnb_gram_noise_level(_dense_code(dtype)))


def _project_lowp(A: torch.Tensor, V: torch.Tensor, inner: int) -> torch.Tensor:
    """project_bf16 / project_f16 / project_f8 on a CUDA matrix of their dtype and a float32 V."""
    project, lead = _TC_LOWP[A.dtype][2:]
    A, V = A.contiguous(), V.contiguous()
    rows, n = A.shape
    r = V.shape[1]
    out = torch.empty(rows * r if inner > 0 else (rows, r), dtype=torch.float32, device=A.device)
    L = lib()
    ws = _workspace(L.tnb_project_tc_workspace_bytes(n, r), A.device)
    with torch.cuda.device(A.device):
        check(getattr(L, project)(*lead, _ptr(A), rows, n, _ptr(V), r, int(inner), _ptr(out), _ptr(ws), ws.numel(),
                                  _stream()))
    return out


def project_bf16(A: torch.Tensor, V: torch.Tensor, inner: int = 0) -> torch.Tensor:
    """A (rows x n, bfloat16) @ V (n x r, float32) at fp32 accuracy on the tensor cores, float32 result.  inner > 0
    writes it K-blocked like project_kblocked_out (returned flat)."""
    _require_cuda(A, "project_bf16")
    assert A.dtype == torch.bfloat16 and V.dtype == torch.float32
    return _project_lowp(A, V, inner)


def project_f16(A: torch.Tensor, V: torch.Tensor, inner: int = 0) -> torch.Tensor:
    """A (rows x n, float16) @ V (n x r, float32) at fp32 accuracy on the tensor cores (two fp16 terms of V scaled per
    column by a power of two), float32 result.  inner > 0 writes it K-blocked like project_kblocked_out (returned
    flat)."""
    _require_cuda(A, "project_f16")
    assert A.dtype == torch.float16 and V.dtype == torch.float32
    return _project_lowp(A, V, inner)


def project_f8(A: torch.Tensor, V: torch.Tensor, inner: int = 0) -> torch.Tensor:
    """A (rows x n, float8 e4m3fn or e5m2) @ V (n x r, float32) at fp32 accuracy on the tensor cores (A widened to fp16
    in registers, the two scaled fp16 terms of V of project_f16), float32 result.  inner > 0 writes it K-blocked like
    project_kblocked_out (returned flat)."""
    _require_cuda(A, "project_f8")
    assert A.dtype in _DT_F8 and V.dtype == torch.float32
    return _project_lowp(A, V, inner)


def atb_tensorcore(A: torch.Tensor, B: torch.Tensor, alpha: float = 1.0, D: Optional[torch.Tensor] = None,
                   beta: float = 0.0) -> torch.Tensor:
    """alpha * A^T B + beta * D on the tensor-core kernel (A: K x m, B: K x n, fp32)."""
    _require_cuda(A, "atb_tensorcore")
    A, B = A.contiguous(), B.contiguous()
    K, m = A.shape
    n = B.shape[1]
    L = lib()
    ws = _workspace(L.tnb_atb_tc_workspace_bytes(K, m, n), A.device)
    out = torch.empty(m, n, dtype=torch.float32, device=A.device)
    with torch.cuda.device(A.device):
        check(L.tnb_atb_tc_f32(_ptr(A), K, m, _ptr(B), n, _ptr(out), float(alpha), _ptr(D), float(beta), _ptr(ws),
                               ws.numel(), _stream()))
    return out


def cheb_filter(G: torch.Tensor, Y0: torch.Tensor, a, bc, g) -> torch.Tensor:
    """len(a) three-term filter products Y_s = a_s G Y_{s-1} + bc_s Y_{s-1} + g_s Y_{s-2} as one resident
    cluster kernel (csrc/cheb_filter.cuh); fp32 blocks, TF32 products."""
    _require_cuda(G, "cheb_filter")
    n, b = Y0.shape
    steps = len(a)
    bufs = [Y0.contiguous().clone(), torch.empty_like(Y0), torch.empty_like(Y0)]
    ws = _workspace(lib().tnb_cheb_filter_workspace_bytes(n, b), G.device)
    fa, fb, fg = ((C.c_float * steps)(*[float(v) for v in x]) for x in (a, bc, g))
    with torch.cuda.device(G.device):
        check(lib().tnb_cheb_filter_f32(_ptr(G.contiguous()), n, b, _ptr(bufs[0]), _ptr(bufs[1]), _ptr(bufs[2]), steps,
                                        fa, fb, fg, _ptr(ws), ws.numel(), _stream()))
    return bufs[steps % 3]


def project(A: torch.Tensor, V: torch.Tensor, tensorcore: bool = False) -> torch.Tensor:
    _require_cuda(A, "project")
    A, V = A.contiguous(), V.contiguous()
    rows, n = A.shape
    assert V.shape[0] == n and V.dtype == A.dtype
    r = V.shape[1]
    Cc = torch.empty(rows, r, dtype=A.dtype, device=A.device)
    if tensorcore:
        L = lib()
        wsb = L.tnb_project_tc_workspace_bytes(n, r)
        if A.dtype != torch.float32:
            check(_lib.ERR_UNSUPPORTED)
        ws = _workspace(wsb, A.device)
        with torch.cuda.device(A.device):
            check(L.tnb_project_tc_f32(_ptr(A), rows, n, _ptr(V), r, _ptr(Cc), _ptr(ws), ws.numel(), _stream()))
        return Cc
    with torch.cuda.device(A.device):
        check(lib().tnb_project(_dtype_code(A), _ptr(A), rows, n, _ptr(V), r, _ptr(Cc), _stream()))
    return Cc


def project_kblocked_out(A: torch.Tensor, V: torch.Tensor, inner: int) -> torch.Tensor:
    """project(A, V, tensorcore=True) written K-blocked as the (rows/inner) x (inner*r) matrix whose row a holds rows
    a*inner .. a*inner+inner-1 of the product (the sweep's carry for a next step with I = inner); returned flat."""
    _require_cuda(A, "project_kblocked_out")
    A, V = A.contiguous(), V.contiguous()
    rows, n = A.shape
    r = V.shape[1]
    out = torch.empty(rows * r, dtype=torch.float32, device=A.device)
    L = lib()
    wsb = L.tnb_project_tc_workspace_bytes(n, r)
    if A.dtype != torch.float32:
        check(_lib.ERR_UNSUPPORTED)
    ws = _workspace(wsb, A.device)
    with torch.cuda.device(A.device):
        check(L.tnb_project_tc_kblocked_out_f32(_ptr(A), rows, n, _ptr(V), r, int(inner), _ptr(out), _ptr(ws), ws.numel(),
                                                _stream()))
    return out


def project_kblocked_in(B: torch.Tensor, rows: int, V: torch.Tensor) -> torch.Tensor:
    """project(A, V, tensorcore=True) for the (rows x n) fp32 matrix A stored K-blocked in B (to_kblocked)."""
    _require_cuda(B, "project_kblocked_in")
    V = V.contiguous()
    n, r = V.shape
    assert B.dtype == torch.float32 and B.is_contiguous() and B.numel() == rows * n
    Cc = torch.empty(rows, r, dtype=torch.float32, device=B.device)
    L = lib()
    ws = _workspace(L.tnb_project_tc_workspace_bytes(n, r), B.device)
    with torch.cuda.device(B.device):
        check(L.tnb_project_tc_kblocked_in_f32(_ptr(B), rows, n, _ptr(V), r, _ptr(Cc), _ptr(ws), ws.numel(), _stream()))
    return Cc


def eigh_jacobi(G: torch.Tensor, return_sweeps: bool = False):
    _require_cuda(G, "eigh_jacobi")
    G = G.contiguous().double()
    n = G.shape[0]
    w = torch.empty(n, dtype=torch.float64, device=G.device)
    V = torch.empty(n, n, dtype=torch.float64, device=G.device)
    L = lib()
    ws = _workspace(L.tnb_eigh_workspace_bytes(n), G.device)
    with torch.cuda.device(G.device):
        check(L.tnb_eigh_jacobi(_ptr(G), n, _ptr(w), _ptr(V), _ptr(ws), ws.numel(), _stream()))
    if return_sweeps:  # the kernel leaves its sweep count right behind the (256-byte aligned) scratch matrices
        npad = n + (n & 1)
        off = (2 * npad * (npad + 8) * 8 + 255) // 256 * 256
        return w, V, int(ws[off: off + 4].view(torch.int32).item())
    return w, V


def eig_topk(G: torch.Tensor, k: int, b: int = 0, tol: float = 1e-6):
    _require_cuda(G, "eig_topk")
    G = G.contiguous().double()
    n = G.shape[0]
    L = lib()
    wsb = L.tnb_eig_topk_workspace_bytes(n, k, b)
    ws = _ws(wsb, G.device)
    bb = b if b > 0 else min(n, min(256, max(2 * k, k + 16)))
    w = torch.empty(bb, dtype=torch.float64, device=G.device)
    V = torch.empty(n, bb, dtype=torch.float64, device=G.device)
    info = (C.c_double * 4)()
    with torch.cuda.device(G.device):
        check(L.tnb_eig_topk(_ptr(G), n, k, b, float(tol), _ptr(w), _ptr(V), _ptr(ws), ws.numel(), info, _stream()))
    return w, V, dict(products=int(info[0]), outer=int(info[1]), converged=int(info[2]))


def tt_relative_error(data: torch.Tensor, cores: Sequence[torch.Tensor]) -> float:
    """‖data − TT(cores)‖_F / ‖data‖_F, fp64 accumulation on the device (metrics.py:135-151).  bfloat16, float16 and
    float8 data take float32 cores (what ttsvd returns for them)."""
    _require_cuda(data, "tt_relative_error")
    data = data.contiguous()
    cores = [c.contiguous() for c in cores]
    N = data.dim()
    code = _dense_code(data.dtype)
    ranks = _tt_ranks(cores, "tt_relative_error")
    if data.dtype in _DT_LOW and cores[0].dtype != torch.float32:
        raise ValueError(f"tt_relative_error: {str(data.dtype).replace('torch.', '')} data needs float32 cores")
    if len(cores) != N or [c.shape[1] for c in cores] != list(data.shape):
        raise ValueError("tt_relative_error: the cores' mode sizes must match data.shape")
    L = lib()
    sh, rk = i64(list(data.shape)), i32(ranks)
    ws = _workspace(L.tnb_tt_relative_error_workspace_bytes(code, N, sh, rk), data.device)
    ptrs = (C.c_void_p * N)(*[c.data_ptr() for c in cores])
    res = (C.c_double * 1)()
    with torch.cuda.device(data.device):
        check(L.tnb_tt_relative_error(code, _ptr(data), ptrs, N, sh, rk, _ptr(ws), ws.numel(), res, _stream()))
    return float(res[0])


_DT_OUT = {torch.float32: _lib.TNB_F32, torch.float64: _lib.TNB_F64, torch.bfloat16: _lib.TNB_BF16, torch.float16: _lib.TNB_F16}


def tt_decompress(cores: Sequence[torch.Tensor], dtype: Optional[torch.dtype] = None,
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The dense tensor of TT cores [r, I, r'] (one dtype, one CUDA device, boundary ranks 1) in one library call
    (tnb_tt_decompress): stream-ordered, no host synchronisation.  `dtype` defaults to the cores' dtype; float32 cores
    also decompress to bfloat16 or float16 (the float32 result rounded once).  `out`: a preallocated contiguous tensor of
    the result's shape and dtype."""
    cores = list(cores)
    ranks = _tt_ranks(cores, "tt_decompress", boundary=True)
    c0 = cores[0]
    if any(c.requires_grad for c in cores):
        raise ValueError("tt_decompress: cores that require grad are not supported (use Tensor.torch() without arguments)")
    dtype = c0.dtype if dtype is None else dtype
    shape = [c.shape[1] for c in cores]
    if out is None:
        out = torch.empty(shape, dtype=dtype, device=c0.device)
    elif list(out.shape) != shape or out.dtype != dtype or out.device != c0.device or not out.is_contiguous():
        raise ValueError(f"tt_decompress: out must be a contiguous {dtype} tensor of shape {shape} on {c0.device}")
    code, ocode = _dtype_code(c0), _DT_OUT.get(dtype, -1)
    cores = [c.contiguous() for c in cores]
    N = len(cores)
    L = lib()
    sh, rk = i64(shape), i32(ranks)
    wsb = L.tnb_tt_decompress_workspace_bytes(code, ocode, N, sh, rk)
    ws = _ws(wsb, c0.device)
    ptrs = (C.c_void_p * N)(*[c.data_ptr() for c in cores])
    with torch.cuda.device(c0.device):
        check(L.tnb_tt_decompress(code, ocode, ptrs, N, sh, rk, _ptr(out), _ptr(ws), wsb, _stream()))
    return out


def _gather_key(idx, shape, first: int, last: int, device, check: bool) -> torch.Tensor:
    """idx as a contiguous int64 [P, last - first] tensor on `device`.  With `check`, an index outside [0, I_k) raises
    IndexError before anything is launched: a host key is checked on the host, a device key by one reduction and one
    host synchronisation."""
    M = last - first
    on_device = isinstance(idx, torch.Tensor) and idx.is_cuda
    if isinstance(idx, torch.Tensor):
        if idx.dtype not in (torch.int32, torch.int64):
            raise ValueError(f"tt_gather: indices must be int32 or int64, got {idx.dtype}")
        key = idx
    else:
        key = torch.as_tensor(np.asarray(idx))
        if key.dtype not in (torch.int32, torch.int64):
            raise ValueError(f"tt_gather: indices must be int32 or int64, got {key.dtype}")
    if key.dim() == 1 and M == 1:
        key = key[:, None]
    if key.dim() != 2 or key.shape[1] != M or key.shape[0] < 1:
        raise ValueError(f"tt_gather: indices must be [P >= 1, {M}], got {list(key.shape)}")
    if check:
        hi = torch.tensor(list(shape[first:last]), dtype=torch.int64, device=key.device)
        bad = (key < 0) | (key >= hi)
        if bad.any().item() if on_device else bool(bad.any()):
            p, m = (int(v) for v in bad.nonzero()[0])
            raise IndexError(f"index {int(key[p, m])} is out of bounds for mode {first + m} of size {shape[first + m]}")
    if on_device and key.device != device:
        raise ValueError("tt_gather: indices must be on the host or on the cores' device")
    return key.to(device=device, dtype=torch.int64).contiguous()


def tt_gather_batch(trains, idx, first: int = 0, last: Optional[int] = None, check: bool = True) -> torch.Tensor:
    """Entries of B tensor trains of one shape at P multi-indices over the modes [first, last), from one library call
    (tnb_tt_gather) that forms nothing but each point's running state: out[t, a, p, b] =
    (G_first[:, i_p0, :] ... G_{last-1}[:, i_p(M-1), :])[a, b], as a [B, r_first, P, r_last] tensor in the cores' dtype
    (float32 or float64).  The trains may differ in their inner ranks but not in r_first and r_last.  `idx` is
    [P, last - first] int32 or int64, on the host (uploaded) or on the cores' device.  With `check=True` an index outside
    [0, I_k) raises IndexError before anything launches; for a device key that costs one reduction and one host
    synchronisation (the reference moves every key to the host).  With `check=False` the call has no host
    synchronisation, and an out-of-range index gives NaN for its point.
    When grad mode is on and a core of the range requires grad, the result is differentiable with respect to the
    range's cores: the backward is one library call (tnb_tt_gather_grad) on the key the forward validated, without a
    second check or a host synchronisation; a point with an out-of-range index (check=False) adds nothing to any
    gradient.  It is differentiable once: a double backward raises."""
    trains = [list(t) for t in trains]
    if not trains or not trains[0]:
        raise ValueError("tt_gather: no trains")
    N = len(trains[0])
    last = N if last is None else int(last)
    first = int(first)
    if not 0 <= first < last <= N:
        raise ValueError(f"tt_gather: mode range [{first}, {last}) is not inside [0, {N})")
    shape, ranks = None, []
    for cores in trains:
        if len(cores) != N:
            raise ValueError(f"tt_gather: every train must be {N} 3-D cores [r, I, r']")
        ranks += _tt_ranks(cores, "tt_gather")
        sh = [c.shape[1] for c in cores]
        if shape is None:
            shape = sh
        elif sh != shape:
            raise ValueError(f"tt_gather: every train must have the shape {shape}, got {sh}")
    R = N + 1
    ra, rl = ranks[first], ranks[last]
    if any(ranks[t * R + first] != ra or ranks[t * R + last] != rl for t in range(len(trains))):
        raise ValueError("tt_gather: every train must have the same ranks at the ends of the range")
    c0 = trains[0][first]
    allc = [c for cores in trains for c in cores[first:last]]
    if any(c.device != c0.device for c in allc):
        raise ValueError("tt_gather: cores must share one CUDA device")
    if any(c.dtype != c0.dtype for c in allc) or c0.dtype not in _DT:
        raise ValueError("tt_gather: cores must all be float32 or all float64")
    key = _gather_key(idx, shape, first, last, c0.device, check)
    plan = _GatherPlan(len(trains), N, shape, ranks, first, last, key)
    if torch.is_grad_enabled() and any(c.requires_grad for c in allc):
        return _TtGather.apply(plan, *allc)
    return plan.forward([c for cores in trains for c in cores[first:last]])


class _GatherPlan:
    """One tt_gather call's shapes and validated device key, shared by its forward and its backward."""

    def __init__(self, B, N, shape, ranks, first, last, key):
        self.B, self.N, self.shape, self.ranks, self.first, self.last, self.key = B, N, shape, ranks, first, last, key
        self.P = key.shape[0]

    def _ptrs(self, range_tensors):
        """The B x N pointer table of the range's tensors (B x (last - first), train-major); null outside the range."""
        M = self.last - self.first
        table = [None] * (self.B * self.N)
        for t in range(self.B):
            for m in range(M):
                table[t * self.N + self.first + m] = range_tensors[t * M + m].data_ptr()
        return (C.c_void_p * len(table))(*table)

    def forward(self, cores):
        c0 = cores[0]
        cs = [c.contiguous() for c in cores]
        code, L = _DT[c0.dtype], lib()
        sh, rk = i64(self.shape), i32(self.ranks)
        B, N, first, last, P = self.B, self.N, self.first, self.last, self.P
        wsb = L.tnb_tt_gather_workspace_bytes(code, B, N, sh, rk, first, last, P)
        ws = _workspace(wsb, c0.device)
        out = torch.empty(B, self.ranks[first], P, self.ranks[last], dtype=c0.dtype, device=c0.device)
        with torch.cuda.device(c0.device):
            _lib.check(L.tnb_tt_gather(code, self._ptrs(cs), B, N, sh, rk, first, last, _ptr(self.key), P, _ptr(out),
                                       _ptr(ws), wsb, _stream()))
        return out

    def backward(self, cores, grad_out):
        """The gradients of the range's cores (tnb_tt_gather_grad), in the order of `cores`."""
        c0 = cores[0]
        cs = [c.contiguous() for c in cores]
        gout = grad_out.to(c0.dtype).contiguous()
        grads = [torch.empty(c.shape, dtype=c.dtype, device=c.device) for c in cs]
        code, L = _DT[c0.dtype], lib()
        sh, rk = i64(self.shape), i32(self.ranks)
        B, N, first, last, P = self.B, self.N, self.first, self.last, self.P
        wsb = L.tnb_tt_gather_grad_workspace_bytes(code, B, N, sh, rk, first, last, P)
        ws = _workspace(wsb, c0.device)
        with torch.cuda.device(c0.device):
            _lib.check(L.tnb_tt_gather_grad(code, self._ptrs(cs), B, N, sh, rk, first, last, _ptr(self.key), P,
                                            _ptr(gout), self._ptrs(grads), _ptr(ws), wsb, _stream()))
        return grads


class _TtGather(torch.autograd.Function):
    """tt_gather_batch under autograd: the forward is one tnb_tt_gather call, the backward one tnb_tt_gather_grad
    call on the key the forward validated (no second check, no host synchronisation)."""

    @staticmethod
    def forward(ctx, plan, *cores):
        ctx.plan = plan
        ctx.save_for_backward(*cores)
        return plan.forward(list(cores))

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        cores = ctx.saved_tensors
        grads = ctx.plan.backward(list(cores), grad_out)
        return (None,) + tuple(g if need else None for g, need in zip(grads, ctx.needs_input_grad[1:]))


def tt_gather(cores: Sequence[torch.Tensor], idx, first: int = 0, last: Optional[int] = None,
              check: bool = True) -> torch.Tensor:
    """Entries of one tensor train at P multi-indices over the modes [first, last) as [r_first, P, r_last]
    (tt_gather_batch with one train).  For the full range of a train with boundary ranks 1, out[0, :, 0] are the values
    tntorch's t[Xs].torch() returns."""
    return tt_gather_batch([cores], idx, first, last, check)[0]


def tt_multiply(cores: Sequence[torch.Tensor], X: torch.Tensor) -> torch.Tensor:
    """Y = X.reshape(-1, I) @ M for the TT-matrix M of cores [r_k, i_k, o_k, r_{k+1}] (one dtype, one CUDA device,
    boundary ranks 1), in one library call (tnb_tt_multiply) that never forms M: stream-ordered, no host
    synchronisation.  Returns a fresh [b, O] tensor in the cores' dtype (I = prod i_k, O = prod o_k).  X must have at
    least two dimensions and the cores' dtype and device; it is read in place when it is contiguous."""
    cores = list(cores)
    if cores and any(c.dim() == 5 for c in cores):
        raise NotImplementedError("tt_multiply: batched TT-matrices (5-D cores) are not supported")
    if not cores or any(c.dim() != 4 for c in cores):
        raise ValueError("tt_multiply: cores must be 4-D tensors [r, i, o, r']")
    c0 = cores[0]
    _require_cuda(c0, "tt_multiply")
    if any(c.dtype != c0.dtype or c.device != c0.device for c in cores):
        raise ValueError("tt_multiply: cores must share one dtype and one device")
    ranks = [c0.shape[0]] + [c.shape[3] for c in cores]
    if ranks[0] != 1 or ranks[-1] != 1:
        raise ValueError(f"tt_multiply: boundary ranks must be 1, got {ranks[0]} and {ranks[-1]}")
    if any(a.shape[3] != b.shape[0] for a, b in zip(cores[:-1], cores[1:])):
        raise ValueError("tt_multiply: core ranks do not match")
    assert X.dim() > 1
    if X.dtype != c0.dtype:
        raise RuntimeError(f"tt_multiply: X is {X.dtype} but the cores are {c0.dtype}")
    if X.device != c0.device:
        raise RuntimeError(f"tt_multiply: X is on {X.device} but the cores are on {c0.device}")
    code = _dtype_code(c0)
    idims, odims = [c.shape[1] for c in cores], [c.shape[2] for c in cores]
    I = 1
    for n in idims:
        I *= n
    O = 1
    for n in odims:
        O *= n
    X = X.reshape(-1, I).contiguous()
    b = X.shape[0]
    Y = torch.empty(b, O, dtype=c0.dtype, device=c0.device)
    if b == 0:
        return Y
    cores = [c.contiguous() for c in cores]
    d = len(cores)
    L = lib()
    ii, oo, rk = i64(idims), i64(odims), i32(ranks)
    wsb = L.tnb_tt_multiply_workspace_bytes(code, d, ii, oo, rk, b)
    ws = _workspace(wsb, c0.device)
    ptrs = (C.c_void_p * d)(*[c.data_ptr() for c in cores])
    with torch.cuda.device(c0.device):
        check(L.tnb_tt_multiply(code, ptrs, d, ii, oo, rk, _ptr(X), b, _ptr(Y), _ptr(ws), wsb, _stream()))
    return Y


def tt_dot_batch(pairs) -> torch.Tensor:
    """[<a_p, b_p> for each pair (a_cores, b_cores)] as a [P] float64 tensor, from one library call (tnb_tt_dot) that
    forms neither tensor: stream-ordered, no host synchronisation.  Every train has the same shape (ValueError
    otherwise) and its own ranks; boundary ranks 1.  The arithmetic is fp64: float32 cores are widened exactly as they
    are read, bfloat16 and float16 cores are converted to float32 first (exactly), and a call with any other floating
    type among its cores reads them all as float64.  A pair may be (cores, cores): a squared norm."""
    pairs = [(list(a), list(b)) for a, b in pairs]
    if not pairs:
        raise ValueError("tt_dot_batch: no pairs")
    shape = None
    ranks_a, ranks_b = [], []
    for a, b in pairs:
        if len(a) != len(b):
            raise NotImplementedError(f"tt_dot: trains of unequal length ({len(a)} and {len(b)} cores) are not supported")
        for cores, rk in ((a, ranks_a), (b, ranks_b)):
            rk += _tt_ranks(cores, "tt_dot", boundary=True, one_dtype=False)
            sh = [c.shape[1] for c in cores]
            if shape is None:
                shape = sh
            elif sh != shape:
                raise ValueError(f"tt_dot: every train must have the shape {shape}, got {sh}")
    c0 = pairs[0][0][0]
    allc = [c for a, b in pairs for c in a + b]
    if any(c.device != c0.device for c in allc):
        raise ValueError("tt_dot: cores must share one CUDA device")
    if any(c.requires_grad for c in allc):
        raise ValueError("tt_dot: cores that require grad are not supported")
    dts = {c.dtype for c in allc}
    if any(not dt.is_floating_point for dt in dts):
        raise ValueError(f"tt_dot: floating-point cores expected, got {sorted(map(str, dts))}")
    dt = torch.float32 if dts <= {torch.float32, torch.bfloat16, torch.float16} else torch.float64

    ca, cb = [], []
    for a, b in pairs:
        a2 = [c.to(dt).contiguous() for c in a]
        ca += a2
        cb += a2 if all(x is y for x, y in zip(a, b)) else [c.to(dt).contiguous() for c in b]
    P, N = len(pairs), len(shape)
    code = _DT[dt]
    L = lib()
    sh, ra, rb = i64(shape), i32(ranks_a), i32(ranks_b)
    wsb = L.tnb_tt_dot_workspace_bytes(code, P, N, sh, ra, rb)
    ws = _workspace(wsb, c0.device)
    out = torch.empty(P, dtype=torch.float64, device=c0.device)
    pa = (C.c_void_p * (P * N))(*[c.data_ptr() for c in ca])
    pb = (C.c_void_p * (P * N))(*[c.data_ptr() for c in cb])
    with torch.cuda.device(c0.device):
        check(L.tnb_tt_dot(code, pa, pb, P, N, sh, ra, rb, _ptr(out), _ptr(ws), wsb, _stream()))
    return out


def tt_dot(a_cores: Sequence[torch.Tensor], b_cores: Sequence[torch.Tensor]) -> torch.Tensor:
    """<a, b> of two tensor trains of one shape as a 0-d float64 tensor on their device (tt_dot_batch with one pair)."""
    return tt_dot_batch([(a_cores, b_cores)])[0]

