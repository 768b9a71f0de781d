"""-m gpu: TT rounding path by path against the fp64 oracle (oracle.tt_oracle.round_tt, NumPy SVD).

The rounding dispatcher (csrc/round_impl.cuh, tt_round_any) sends a tensor to one of several paths: the speculative
sweeps (one synchronisation; eligible with a rank cap on every bond, no eps budget, full-rank-shaped left unfoldings and
input ranks <= 104), the host-driven sweeps (Cholesky-QR per core, or an eigen-decomposition for a short core or a
Cholesky breakdown), and, for a batch, the in-flight driver that redoes each rejected tensor host-driven.  Every case
here names the path it must take (read from tt_round_batch(..., return_info=True)["speculative"]) and checks, on the
same core values in fp64:
  (a) the output ranks equal the oracle's;
  (b) |relerr_lib - relerr_oracle| against the dense fp64 input;
  (c) cores 1..N-1 have orthonormal right unfoldings (see U64 below for the bound);
  (d) the input cores are unchanged;
  (e) the path taken;
  (f) speculate=False (the host-driven sweeps) gives the same ranks and relative error.
Every input is small enough to reconstruct densely (<= 2^21 elements), so errors are measured directly.
Run with -s to see the measured deviations."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import cases
from oracle import tt_oracle as orc

pytestmark = pytest.mark.gpu

DTYPES = [torch.float64, torch.float32]
# relerr: (b); orth: (c); paths: (f); exact: relerr of an untruncated rounding
TOL = {
    torch.float64: dict(relerr=1e-8, orth=1e-10, paths=1e-12, exact=1e-12),
    torch.float32: dict(relerr=1e-5, orth=1e-5, paths=1e-6, exact=1e-6),
}
NP_DTYPE = {torch.float64: np.float64, torch.float32: np.float32}
SHAPE5 = (12,) * 5


# ---------------------------------------------------------------------------------------------------- inputs
def _short_last(cores, keep, seed):
    """Replace the last core (r x I x 1) by B (r x keep) C (keep x I), B's rows past `keep` zero.  Phase A carries an
    upper-triangular factor into this core, so the last step's unfolding has exactly zero rows past `keep` and its
    Gram exactly zero eigenvalues: the rank rule returns `keep` below any cap above it, as the reference's SVD does.
    (With a dense B the null space sits at the fp64 Gram's rounding level, ~1e-16 of its norm, which the rank rule
    cannot tell from signal under the default eps budget -- the documented Gram-vs-SVD deviation of DESIGN.md.)"""
    rng = np.random.default_rng(seed)
    r, I, _ = cores[-1].shape
    B = np.zeros((r, keep))
    B[:keep] = rng.standard_normal((keep, keep))
    cores = list(cores)
    cores[-1] = (B @ rng.standard_normal((keep, I))).reshape(r, I, 1)
    return cores


def _zero_core(cores, k):
    cores = list(cores)
    cores[k] = np.zeros_like(cores[k])
    return cores


def _doubled(shape, rank, seed):
    """t + t as block cores: every left unfolding has exactly collinear column pairs."""
    return cases.make_tt(dict(shape=shape, rank=rank, seed=seed, doubled=True))


def _graded(seed):
    """(16,)^5 rank 12 whose first left unfolding has singular values logspace(0, -4) (kappa = 1e4: the diagonally
    scaled Cholesky pivots stay near 1e-8, above the 1e-11 breakdown test); the other cores are Gaussian, so every later
    absorbed unfolding has kappa <= ~2e4."""
    shape, r = (16,) * 5, 12
    rng = np.random.default_rng(seed)
    cores = cases.random_tt(shape, r, seed)
    U, _ = np.linalg.qr(rng.standard_normal((shape[0], r)))
    W, _ = np.linalg.qr(rng.standard_normal((r, r)))
    cores[0] = ((U * np.logspace(0, -4, r)) @ W.T).reshape(1, shape[0], r)
    return cores


def _gapped(seed):
    """A rank-4 TT plus 1e-4 times a rank-3 TT (block cores, rank 7): a clear gap in every bond's spectrum."""
    a = cases.random_tt(SHAPE5, 4, seed)
    b = cases.random_tt(SHAPE5, 3, seed + 1)
    return _block_sum([a, b], [1.0, 1e-4])


def _block_sum(operands, alpha):
    """sum_k alpha_k T_k as block TT cores (Tensor.__add__: the scalar goes into the first core)."""
    N = len(operands[0])
    out = []
    for n in range(N):
        blocks = [op[n] for op in operands]
        if n == 0:
            out.append(np.concatenate([a * c for a, c in zip(alpha, blocks)], axis=2))
        elif n == N - 1:
            out.append(np.concatenate(blocks, axis=0))
        else:
            r0, r1 = sum(c.shape[0] for c in blocks), sum(c.shape[2] for c in blocks)
            z = np.zeros((r0, blocks[0].shape[1], r1))
            i = j = 0
            for c in blocks:
                z[i: i + c.shape[0], :, j: j + c.shape[2]] = c
                i, j = i + c.shape[0], j + c.shape[2]
            out.append(z)
    return out


# name -> input builder and what to expect.  path: 1 speculative, 0 host-driven, None whatever the dispatcher decides.
# orth32=False: fp32 orthonormality is printed, not asserted (kappa = 1e4 in phase A: the fp32 Cholesky-QR factors
# lose orthogonality as roughly u32 * kappa there, above 1e-5, while the rounding error still matches the oracle).
CASES = {
    "accepted_rmax3": dict(make=lambda: cases.random_tt(SHAPE5, 10, 301), rmax=3, path=1),
    "accepted_ragged": dict(make=lambda: cases.random_tt(SHAPE5, 10, 302), rmax=[2, 5, 4, 3], path=1),
    "accepted_untruncated": dict(make=lambda: cases.random_tt(SHAPE5, 10, 303), rmax=16, path=1, exact=True,
                                 ranks=[1, 10, 10, 10, 10, 1]),
    "chol_breakdown": dict(make=lambda: _doubled(SHAPE5, 5, 304), rmax=3, path=0),
    "short_rank": dict(make=lambda: _short_last(cases.random_tt((16, 16, 16), 8, 305), 2, 306), rmax=6, path=0,
                       ranks=[1, 6, 2, 1]),
    "zero_core": dict(make=lambda: _zero_core(cases.random_tt(SHAPE5, 10, 307), 2), rmax=3, path=0, zero=True),
    "graded": dict(make=lambda: _graded(308), rmax=6, path=1, orth32=False),
    "eps_1e-3": dict(make=lambda: _gapped(309), eps=1e-3, rmax=7, path=0, ranks=[1, 4, 4, 4, 4, 1]),
    "eps_1e-8": dict(make=lambda: _gapped(309), eps=1e-8, rmax=7, path=0, ranks=[1, 7, 7, 7, 7, 1]),
    "short_first_core": dict(make=lambda: cases.random_tt((4, 12, 12, 12), 10, 311), rmax=3, path=0),
    # Cholesky with L, L^-1 in shared memory up to 107 columns, global scratch above; speculation up to rank 104
    "rank104": dict(make=lambda: cases.random_tt((128, 6, 6, 128), 104, 312), rmax=20, path=1),
    "rank105": dict(make=lambda: cases.random_tt((128, 6, 6, 128), 105, 313), rmax=20, path=0),
    "rank107": dict(make=lambda: cases.random_tt((128, 6, 6, 128), 107, 314), rmax=20, path=0),
    "rank108": dict(make=lambda: cases.random_tt((128, 6, 6, 128), 108, 315), rmax=20, path=0),
    "rank200": dict(make=lambda: cases.random_tt((256, 4, 256), 200, 316), rmax=20, path=0),
    "tiny_N2": dict(make=lambda: cases.random_tt((12, 12), 5, 317), rmax=3, path=None),
    "tiny_I1": dict(make=lambda: cases.random_tt((6, 1, 7, 5), 4, 318), rmax=3, path=None),
    "tiny_rmax1": dict(make=lambda: cases.random_tt((12,) * 4, 5, 319), rmax=1, path=None),
    "tiny_N1": dict(make=lambda: cases.random_tt((12,), [], 320), rmax=None, path=None),
}
RANK_EDGES = ["rank104", "rank105", "rank107", "rank108", "rank200"]


# ---------------------------------------------------------------------------------------------------- helpers
def _as_input(cores64, dtype):
    """(device cores in `dtype`, the same values as fp64 NumPy cores)."""
    cast = [np.ascontiguousarray(c, dtype=NP_DTYPE[dtype]) for c in cores64]
    return [torch.as_tensor(c).cuda() for c in cast], [c.astype(np.float64) for c in cast]


def _host(cores):
    return [c.detach().cpu().numpy().astype(np.float64) for c in cores]


def _ranks(cores):
    return [1] + [int(c.shape[2]) for c in cores]


def _relerr(dense, cores):
    return float(np.linalg.norm(dense - orc.tt_reconstruct(cores)) / np.linalg.norm(dense))


def _orth(cores):
    """max |M M^T - I| over the right unfoldings M of cores 1..N-1 (0 when N = 1)."""
    dev = 0.0
    for c in cores[1:]:
        M = c.reshape(c.shape[0], -1)
        dev = max(dev, float(np.abs(M @ M.T - np.eye(M.shape[0])).max()))
    return dev


def _kept_kappa(cores):
    """max over the bonds of s_1 / s_r, the spread of the singular values a rounded TT keeps (cores 1..N-1 of the
    oracle's result have orthonormal right unfoldings, so a bond's singular values are its left part's)."""
    kappa, f = 1.0, np.ones((1, 1))
    for c in cores[:-1]:
        f = (f @ c.reshape(c.shape[0], -1)).reshape(-1, c.shape[2])
        s = np.linalg.svd(f, compute_uv=False)
        kappa = max(kappa, s[0] / s[-1])
    return kappa


# The library truncates from the Gram matrix G = M M^T of each unfolding: the kept rows are diag(1/s) U^T M with U
# from a backward-stable eigensolver, U^T G U = diag(s^2) + E with |E| ~ u * s_1^2, so their Gram deviates from I by
# E_ij / (s_i s_j) <= u * (s_1 / s_r)^2 (the reference's SVD: u).  1e-10 holds while the kept spread s_1 / s_r stays
# below ~700; an eps budget that keeps directions 1e-4 below the top (eps_1e-8: spread 6e4, 7e-8 measured on an H100)
# is bounded by u * spread^2 instead.
U64 = float(np.finfo(np.float64).eps) / 2


def _unchanged(dev, before):
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(dev, before)), "the input cores were modified"


def _check_against_oracle(label, dtype, dense, ref, results, zero=False, exact=False, orth=True):
    """(a) (b) (c) for every result in `results` (name -> fp64 cores), (f) between them; returns the deviations."""
    tol = TOL[dtype]
    for name, out in results.items():
        assert _ranks(out) == _ranks(ref), (label, name, _ranks(out), _ranks(ref))
    if zero:
        assert not np.any(orc.tt_reconstruct(ref)), "oracle: a zero tensor rounds to zero"
        for name, out in results.items():
            assert not np.any(orc.tt_reconstruct(out)), (label, name, "does not reconstruct to exactly zero")
        print(f"{label}: ranks {_ranks(ref)}, zero output")
        return {}
    e_ref = _relerr(dense, ref)
    errs = {name: _relerr(dense, out) for name, out in results.items()}
    dev = dict(relerr=max(abs(e - e_ref) for e in errs.values()),
               paths=max(errs.values()) - min(errs.values()),
               orth=max(_orth(out) for out in results.values()))
    tol = dict(tol, orth=max(tol["orth"], U64 * _kept_kappa(ref) ** 2))
    if exact:
        dev["exact"] = max(errs.values())
    print(f"{label}: ranks {_ranks(ref)}, relerr oracle {e_ref:.10f}, "
          + ", ".join(f"{k} {v:.2e} (tol {tol[k]:.1e})" for k, v in dev.items()))
    assert dev["relerr"] <= tol["relerr"], (label, errs, e_ref)
    assert dev["paths"] <= tol["paths"], (label, errs)
    if exact:
        assert dev["exact"] <= tol["exact"], (label, errs)
    if orth:
        assert dev["orth"] <= tol["orth"], (label, dev["orth"])
    return dev


# ---------------------------------------------------------------------------------------------------- single tensors
@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("name", list(CASES))
def test_round_path_matches_oracle(name, dtype):
    from tntorch_b200 import ops

    spec = CASES[name]
    eps, rmax = spec.get("eps", 1e-14), spec["rmax"]
    dev, cores64 = _as_input(spec["make"](), dtype)
    before = [c.clone() for c in dev]
    out, info = ops.tt_round_batch([dev], eps=eps, rmax=rmax, return_info=True)
    host = ops.tt_round(dev, eps=eps, rmax=rmax, speculate=False)
    _, info_off = ops.tt_round_batch([dev], eps=eps, rmax=rmax, speculate=False, return_info=True)
    _unchanged(dev, before)  # (d)
    if spec["path"] is not None:
        assert info["speculative"] == [spec["path"]], info  # (e)
    assert info_off["speculative"] == [0], info_off  # speculate=False never speculates
    ref = orc.round_tt([c.copy() for c in cores64], eps=eps, rmax=rmax)
    if "ranks" in spec:
        assert _ranks(ref) == spec["ranks"], "the input does not have the spectrum this case is built for"
    _check_against_oracle(f"{name} {dtype} path={info['speculative'][0]}", dtype, orc.tt_reconstruct(cores64), ref,
                          dict(dispatch=_host(out[0]), host_driven=_host(host)), zero=spec.get("zero", False),
                          exact=spec.get("exact", False), orth=dtype == torch.float64 or spec.get("orth32", True))


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
def test_input_rank_above_eigensolver_limit_raises(dtype):
    """Input ranks above 256 (JACOBI_MAX_N) are unsupported: an error, not a quiet fallback."""
    from tntorch_b200 import ops

    dev, _ = _as_input(cases.random_tt((300, 2, 300), 257, 321), dtype)
    for speculate in (True, False):
        with pytest.raises(NotImplementedError):
            ops.tt_round(dev, rmax=20, speculate=speculate)
    with pytest.raises(NotImplementedError):
        ops.tt_round_batch([dev, dev], rmax=20)


# ---------------------------------------------------------------------------------------------------- fused sums
SUMS = {
    # a + 2a: exactly collinear blocks, a Cholesky breakdown at the first core
    "collinear": dict(make=lambda: [cases.random_tt(SHAPE5, 5, 330)] * 2, alpha=[1.0, 2.0], rmax=5,
                      ranks=[1, 5, 5, 5, 5, 1]),
    "three": dict(make=lambda: [cases.random_tt((10,) * 4, r, 331 + r) for r in (3, 4, 2)], alpha=[1.0, -0.5, 2.0],
                  rmax=5),
}


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("name", list(SUMS))
def test_fused_sum_round_matches_oracle(name, dtype):
    from tntorch_b200 import ops

    spec = SUMS[name]
    inputs = [_as_input(op, dtype) for op in spec["make"]()]
    dev = [d for d, _ in inputs]
    ops64 = [c for _, c in inputs]
    before = [[c.clone() for c in op] for op in dev]
    out = ops.tt_sum_round(dev, alpha=spec["alpha"], rmax=spec["rmax"])
    host = ops.tt_sum_round(dev, alpha=spec["alpha"], rmax=spec["rmax"], speculate=False)
    for d, b in zip(dev, before):
        _unchanged(d, b)
    dense = sum(a * orc.tt_reconstruct(op) for a, op in zip(spec["alpha"], ops64))
    ref = orc.round_tt(_block_sum(ops64, spec["alpha"]), rmax=spec["rmax"])
    if "ranks" in spec:
        assert _ranks(ref) == spec["ranks"]
    _check_against_oracle(f"sum {name} {dtype}", dtype, dense, ref, dict(dispatch=_host(out), host_driven=_host(host)))


# ---------------------------------------------------------------------------------------------------- batches
def _mixed_batch():
    """Five tensors with the (12,)^5 rank-10 core shapes: accepted, Cholesky breakdown, short last rank, accepted,
    zero core."""
    return [
        cases.random_tt(SHAPE5, 10, 340),
        _doubled(SHAPE5, 5, 341),
        _short_last(cases.random_tt(SHAPE5, 10, 342), 2, 343),
        cases.random_tt(SHAPE5, 10, 344),
        _zero_core(cases.random_tt(SHAPE5, 10, 345), 2),
    ]


MIXED_ZERO = 4


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("eps,expect", [(1e-14, [1, 0, 0, 1, 0]), (1e-3, [0] * 5)], ids=["speculative", "eps_budget"])
def test_mixed_batch_matches_single_calls_and_oracle(eps, expect, dtype):
    """Two tensors in flight over five (workspace slices reused), three of them rejected and redone host-driven in
    slice 0; with an eps budget nothing is eligible and the batch runs one tensor at a time.  Each tensor must equal
    its own B = 1 call and the oracle."""
    from tntorch_b200 import ops

    rmax = 3
    inputs = [_as_input(c, dtype) for c in _mixed_batch()]
    dev = [d for d, _ in inputs]
    before = [[c.clone() for c in d] for d in dev]
    out, info = ops.tt_round_batch(dev, eps=eps, rmax=rmax, inflight=2, return_info=True)
    for d, b in zip(dev, before):
        _unchanged(d, b)
    assert info["speculative"] == expect, info
    for i, (d, cores64) in enumerate(inputs):
        single, _ = ops.tt_round_batch([d], eps=eps, rmax=rmax, return_info=True)
        ref = orc.round_tt([c.copy() for c in cores64], eps=eps, rmax=rmax)
        _check_against_oracle(f"batch[{i}] eps={eps:g} {dtype}", dtype, orc.tt_reconstruct(cores64), ref,
                              dict(batch=_host(out[i]), single=_host(single[0])), zero=i == MIXED_ZERO)


def test_speculate_false_runs_host_driven_on_eligible_input():
    from tntorch_b200 import ops

    dev, _ = _as_input(cases.random_tt(SHAPE5, 10, 301), torch.float64)
    assert ops.tt_round_batch([dev], rmax=3, return_info=True)[1]["speculative"] == [1]
    assert ops.tt_round_batch([dev], rmax=3, speculate=False, return_info=True)[1]["speculative"] == [0]
    assert ops.tt_round_batch([dev] * 3, rmax=3, inflight=2, speculate=False, return_info=True)[1]["speculative"] == [0] * 3


# ---------------------------------------------------------------------------------------------------- buffer bounds
CANARY = 1 << 20


def _guarded(nbytes):
    """A device byte buffer of exactly `nbytes` followed by a 1 MiB canary; returns (buffer, canary pattern)."""
    pattern = ((torch.arange(CANARY, device="cuda") * 151 + 89) % 256).to(torch.uint8)
    buf = torch.empty(nbytes + CANARY, dtype=torch.uint8, device="cuda")
    buf[nbytes:] = pattern
    return buf, pattern


def _intact(buf, nbytes, pattern):
    torch.cuda.synchronize()
    return torch.equal(buf[nbytes:], pattern)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
def test_round_stays_inside_queried_workspace_and_cores(dtype):
    """The workspace is exactly tnb_tt_round_workspace_bytes (the dry-run arena sizes the speculative and the
    host-driven carves separately) and the cores buffer exactly the queried capacity: neither path may write past
    them, on the rank edges and on the mixed batch (speculative, rejected and redone, zero)."""
    from tntorch_b200 import _lib

    L = _lib.lib()
    code = _lib.TNB_F64 if dtype == torch.float64 else _lib.TNB_F32
    esz = 8 if dtype == torch.float64 else 4
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rmax = 20
    for name in RANK_EDGES:
        dev, _ = _as_input(CASES[name]["make"](), dtype)
        N = len(dev)
        sh = _lib.i64([c.shape[1] for c in dev])
        rin = _lib.i32([1] + [c.shape[2] for c in dev])
        rm = _lib.i32([rmax] * (N - 1))
        offs = (C.c_int64 * N)()
        cap = L.tnb_tt_round_cores_capacity(N, sh, rin, rm, offs)
        wsb = L.tnb_tt_round_workspace_bytes(code, N, sh, rin, rm)
        assert cap > 0 and wsb > 0
        ptrs = (C.c_void_p * N)(*[c.data_ptr() for c in dev])
        for flags in (0, _lib.FLAG_NO_SPECULATE):
            ws, pw = _guarded(wsb)
            out, po = _guarded(cap * esz)
            ranks = (C.c_int32 * (N + 1))()
            _lib.check(L.tnb_tt_round(code, ptrs, N, sh, rin, rm, 1e-14, flags, C.c_void_p(ws.data_ptr()), wsb,
                                      C.c_void_p(out.data_ptr()), cap, ranks, stream))
            assert _intact(ws, wsb, pw), (name, flags, "workspace overrun")
            assert _intact(out, cap * esz, po), (name, flags, "cores buffer overrun")
            assert list(ranks) == [1] + [rmax] * (N - 1) + [1], (name, list(ranks))

    batch = [_as_input(c, dtype)[0] for c in _mixed_batch()]
    B, N = len(batch), len(batch[0])
    sh = _lib.i64([c.shape[1] for c in batch[0]])
    rin = _lib.i32([1] + [c.shape[2] for c in batch[0]])
    rm = _lib.i32([3] * (N - 1))
    cap = L.tnb_tt_round_cores_capacity(N, sh, rin, rm, None)
    one = C.c_size_t(0)
    assert L.tnb_tt_round_batch_workspace_bytes(code, B, N, sh, rin, rm, C.byref(one)) > 0
    wsb = one.value * 2  # two slices: two tensors in flight, B = 5 reuses them
    pin = (C.c_void_p * (B * N))(*[c.data_ptr() for cores in batch for c in cores])
    for eps, expect in ((1e-14, [1, 0, 0, 1, 0]), (1e-3, [0] * B)):
        ws, pw = _guarded(wsb)
        outs = [_guarded(cap * esz) for _ in range(B)]
        pout = (C.c_void_p * B)(*[o.data_ptr() for o, _ in outs])
        ranks = (C.c_int32 * (B * (N + 1)))()
        spec = (C.c_int32 * B)()
        _lib.check(L.tnb_tt_round_batch(code, pin, B, N, sh, rin, rm, eps, 0, C.c_void_p(ws.data_ptr()), wsb, pout, cap,
                                        ranks, spec, stream))
        assert list(spec) == expect, list(spec)
        assert _intact(ws, wsb, pw), (eps, "batch workspace overrun")
        for i, (o, po) in enumerate(outs):
            assert _intact(o, cap * esz, po), (eps, i, "batch cores buffer overrun")
