"""-m gpu: the dense TT-SVD of a tensor in host memory (ops.ttsvd_stream / tnb_ttsvd_stream), against ops.ttsvd on the
device copy of the same data: equal ranks, relative error within 1e-6, and reconstructions that agree.  Every input
type, chunk budgets from one chunk to as many as the chunk minimums allow, pinned and pageable sources, the goldens of
the reference, an eps budget, the speculative tail's fallback, the exact-Gram re-stream, the re-solve that needs no
re-stream, the K-blocked carry selected or not, tn.Tensor's routing, and the error from the norm alone."""
import os

import numpy as np
import pytest
import torch

from oracle import cases
import stream_model as sm

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _twin(shape, rank, noise, seed):
    spec = dict(kind="tt_noise", shape=shape, rank=rank, noise=noise, seed=seed)
    return torch.from_numpy(cases.make_dense_big(spec))


def _recon_diff(a, b):
    from tntorch_b200 import ops

    ra, rb = ops.tt_decompress([c.double() for c in a]), ops.tt_decompress([c.double() for c in b])
    return float(torch.linalg.vector_norm(ra - rb) / torch.linalg.vector_norm(rb))


def _compare(X_cpu, rmax, chunk_bytes=None, eps=1e-14, recon_tol=1e-4, pin=False, same_path=True):
    """recon_tol None: a flat spectrum (randn), whose kept subspace is not determined beyond the Gram's rounding; the
    errors still agree."""
    from tntorch_b200 import ops

    src = X_cpu.pin_memory() if pin else X_cpu
    cores, info = ops.ttsvd_stream(src, rmax=rmax, eps=eps, chunk_bytes=chunk_bytes, return_info=True)
    Xd = X_cpu.cuda()
    ref, rinfo = ops.ttsvd(Xd, rmax=rmax, eps=eps, return_info=True)
    assert [int(c.shape[2]) for c in cores] == [int(c.shape[2]) for c in ref]
    e, e_ref = ops.tt_relative_error(Xd, cores), ops.tt_relative_error(Xd, ref)
    assert abs(e - e_ref) <= 1e-6, (e, e_ref, info)
    if recon_tol is not None:
        assert _recon_diff(cores, ref) <= recon_tol, info
    assert abs(info["norm"] - rinfo["norm"]) <= 1e-3 * rinfo["norm"]  # the TF32 Gram's uniform shrink at most
    # the rest of the sweep takes the device call's path: speculative or not, K-blocked carry or not (same_path False:
    # the device call repeated its whole sweep exactly where the stream repeats only step 0)
    assert not same_path or (info["speculative"], info["kblocked_steps"]) == (rinfo["speculative"], rinfo["kblocked_steps"]), (info, rinfo)
    return cores, info, e


def _budgets(X, minimum):
    total = X.numel() * X.element_size()
    return {"one": None, "two": total // 2 + 1, "ragged7": total * 2 // 13, "minimum": minimum}


DTYPES = [torch.float32, torch.float64, torch.bfloat16, torch.float16, torch.float8_e4m3fn, torch.float8_e5m2]


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).replace("torch.", ""))
@pytest.mark.parametrize("budget", ["one", "two", "ragged7", "minimum"])
def test_every_dtype_and_chunk_budget(dtype, budget):
    """32^5 twin at rank 16, scaled to unit RMS (inside the fp8 range).  fp32 projects on the tensor cores (16384-row
    minimum: 64 chunks at a 1-byte budget, blocks of 8 x 32 rows for the K-blocked carry its shape allows); the other
    types take 64 chunks at 1/64 of the tensor."""
    X = _twin((32,) * 5, 16, 1e-2, 301)
    X = (X / X.square().mean().sqrt()).to(dtype)
    total = X.numel() * X.element_size()
    chunk = _budgets(X, 1 if dtype == torch.float32 else total // 64)[budget]
    tol = 1e-9 if dtype == torch.float64 else 1e-4
    _, info, _ = _compare(X, 16, chunk_bytes=chunk, recon_tol=tol)
    f32 = dtype == torch.float32
    want = sm.chunk_plan(32 ** 4, 32, 32 * X.element_size(), chunk, f32, 32 if f32 else 0)[3]
    assert info["chunks"] == want == {"one": 1, "two": 2, "ragged7": 7, "minimum": 64}[budget], info
    assert info["passes"] in (2, 3)


@pytest.mark.parametrize("pin", [False, True])
def test_pinned_and_pageable_sources_agree(pin):
    from tntorch_b200 import ops

    X = _twin((32,) * 5, 16, 1e-2, 302)
    cores, _, _ = _compare(X, 16, chunk_bytes=X.numel() * 4 // 5, pin=pin)
    other = ops.ttsvd_stream(X if pin else X.pin_memory(), rmax=16, chunk_bytes=X.numel() * 4 // 5)
    assert all(torch.equal(a, b) for a, b in zip(cores, other))  # the source's memory kind changes no arithmetic


@pytest.mark.parametrize("rank,kblocked", [(16, 1), (8, 0)])
def test_kblocked_carry_selected_or_not(rank, kblocked):
    """randn 32^5 (a flat spectrum: the speculative tail is accepted) in 64 chunks: at rank 16 the step-0 carry is written
    K-blocked for step 1 as in the device call, at rank 8 (not a multiple of 16) row-major."""
    X = torch.randn((32,) * 5, generator=torch.Generator().manual_seed(303))
    _, info, _ = _compare(X, rank, chunk_bytes=1, recon_tol=None)
    assert info["kblocked_steps"] == kblocked and info["chunks"] == 64 and info["speculative"] == 1, info


@pytest.mark.parametrize("name", [n for n, v in cases.TTSVD_CASES.items() if v.get("ranks_tt") is not None and "shape" in v
                                  and v["kind"] != "zeros" and (lambda s, r: min(r if isinstance(r, int) else r[-1], int(np.prod(s[:-1]))) < s[-1]
                                       and int(np.prod(s[:-1])) >= s[-1])(v["shape"], v["ranks_tt"])])
def test_goldens_of_the_reference(name):
    """the reference's ranks on every rank-capped case the stream takes (tall step 0, a carry smaller than the input)."""
    from tntorch_b200 import ops

    g = np.load(os.path.join(GOLD, "ttsvd.npz"))
    spec = cases.TTSVD_CASES[name]
    X = torch.as_tensor(cases.make_dense(spec))
    for chunk in (None, X.numel() * X.element_size() // 3):
        cores = ops.ttsvd_stream(X, rmax=spec["ranks_tt"], chunk_bytes=chunk)
        assert [1] + [int(c.shape[2]) for c in cores] == list(g[f"{name}/eig/ranks"])
        err = ops.tt_relative_error(X.cuda(), cores)
        # within 1e-5 of the reference, or below it: on smooth_f32_r6 the streamed step 0 lands at 1.9e-7 where the
        # reference's fp32 eigensolver leaves 4.3e-5
        assert err <= float(g[f"{name}/eig/relerr"]) + 1e-5, (name, err)


def test_eps_budget_with_rank_caps():
    """an active eps budget decides ranks under the caps: host-driven sweep after the streamed step 0."""
    X = _twin((24, 20, 16, 28, 32), 6, 1e-3, 304).double()
    cores, info, e = _compare(X, 12, chunk_bytes=X.numel() * 8 // 4, eps=1e-2, recon_tol=1e-9)
    assert info["speculative"] == 0 and e <= 1e-2
    assert [int(c.shape[2]) for c in cores][:-1] != [12] * 4


def test_rank_deficient_tail_falls_back_from_the_kblocked_carry():
    """zero outside X[0]: the step-1... step N-1 Grams keep their caps but the first bond's has exact zero rows, the
    rank rule returns 1 where the cap is 16, the speculative tail is repeated host-driven from the (K-blocked) step-0
    carry, which is rewritten row-major for it; the host tensor is not read again."""
    X = torch.zeros((32,) * 5)
    X[0] = _twin((32,) * 4, 16, 1e-2, 307)
    cores, info, _ = _compare(X, 16, chunk_bytes=X.numel() * 4 // 4)
    assert info["speculative"] == 0 and info["spec_flags"] & 16 and info["passes"] == 2, info
    assert int(cores[0].shape[2]) == 1


def test_rank_deficient_step_zero():
    """the step-0 rule itself returns less than the cap: the rest of the sweep is host-driven, flagged as the
    speculative check would flag it."""
    g = torch.Generator().manual_seed(8)
    X = torch.zeros(16, 16, 16, 64, dtype=torch.float64)
    X[..., :4] = torch.randn(16, 16, 16, 4, generator=g, dtype=torch.float64)
    cores, info, _ = _compare(X, 8, recon_tol=1e-9)
    assert int(cores[2].shape[2]) == 4 and info["speculative"] == 0 and info["spec_flags"] == 16, info


def test_zero_tensor():
    from tntorch_b200 import ops

    cores, info = ops.ttsvd_stream(torch.zeros(8, 9, 64, 16), rmax=4, return_info=True)
    assert [int(c.shape[2]) for c in cores] == [1, 1, 1, 1] and info["norm"] == 0.0 and info["passes"] == 1


def test_rejected_tf32_gram_is_restreamed_exactly():
    """a tail far below the TF32 Gram's noise floor: step 0's tensor-core Gram is rejected and the host tensor is
    streamed a third time through the exact Gram; the result is the device call's and the reference's."""
    from tntorch_b200 import ops

    name = "twin_lownoise_16x5_f32"
    spec = cases.LOWNOISE_CASES[name]
    X = torch.as_tensor(cases.make_dense(spec))
    cores, info, e = _compare(X, spec["ranks_tt"], chunk_bytes=X.numel() * 4 // 3, same_path=False)
    assert info["passes"] == 3 and info["chunks"] == 4, info  # 3 chunks of 21840 rows and one of 16
    g = np.load(os.path.join(GOLD, "lownoise.npz"))
    assert abs(e - float(g[f"{name}/svd/relerr"])) <= 1e-5


def test_rejected_fp32_solve_of_an_exact_gram_is_not_restreamed():
    """fp32 with 12^3 = 1728 step-0 rows, below the tensor-core Gram's 2048: step 0's Gram is exact, and with a
    speculative tail ahead its eigenpairs come from fp32 rotations, whose noise floor the low-noise spectrum (tail ~1e-11
    of the trace) does not clear.  The rejected solve is repeated with fp64 rotations on the same Gram: two passes over
    the host tensor, not three, and one eigensolve more than the device call, whose host-driven repeat solves each step
    once (the stream's tail is rejected the same way and repeated host-driven too)."""
    X = torch.as_tensor(cases.make_dense(dict(kind="tt_noise", shape=(12, 12, 12, 32), rank=6, noise=1e-5, seed=31,
                                              dtype="float32")))
    from tntorch_b200 import ops

    _, info, _ = _compare(X, 6, chunk_bytes=X.numel() * 4 // 3)
    _, rinfo = ops.ttsvd(X.cuda(), rmax=6, eps=1e-14, return_info=True)
    assert info["passes"] == 2 and info["chunks"] == 3 and info["tc_grams"] == 0, info
    assert info["eig_solves"] == rinfo["eig_solves"] + 1 and rinfo["speculative"] == 0, (info, rinfo)


def test_tensor_routing_follows_free_memory(monkeypatch):
    import tntorch_b200 as tnb
    from tntorch_b200 import ops

    X = _twin((32,) * 5, 16, 1e-2, 305)
    calls = []
    real_stream, real_ttsvd = ops.ttsvd_stream, ops.ttsvd
    monkeypatch.setattr(ops, "ttsvd_stream", lambda *a, **k: calls.append("stream") or real_stream(*a, **k))
    monkeypatch.setattr(ops, "ttsvd", lambda *a, **k: calls.append("device") or real_ttsvd(*a, **k))
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (1 << 20, 80 << 30))
    t = tnb.Tensor(X, ranks_tt=16)
    assert calls == ["stream"]
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (70 << 30, 80 << 30))
    t2 = tnb.Tensor(X, ranks_tt=16)
    assert calls == ["stream", "device"]
    assert _recon_diff(t.cores, t2.cores) <= 1e-4
    calls.clear()
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (1 << 20, 80 << 30))
    tnb.Tensor(X.cuda(), ranks_tt=16)  # a device tensor is never streamed
    assert calls == ["device"]


def _from_norm_tol(exact):
    """the norm is the step-0 Gram's trace and core 0 is fp32: ‖T‖² − ‖core_0‖² resolves ~5e-6 of ‖T‖² (measured 2e-6
    on the twin), i.e. 5e-6 / (2 e) in the error e"""
    return 5e-6 / (2 * exact) + 1e-6


def test_relative_error_from_norm():
    from tntorch_b200 import ops

    for X, r in ((torch.randn((32,) * 5, generator=torch.Generator().manual_seed(9)), 16), (_twin((32,) * 5, 16, 1e-2, 306), 16)):
        cores, info = ops.ttsvd_stream(X, rmax=r, return_info=True)
        exact = ops.tt_relative_error(X.cuda(), cores)
        assert abs(ops.tt_relative_error_from_norm(info["norm"], cores) - exact) <= _from_norm_tol(exact), exact


def test_twin_64x5_in_64MiB_chunks_matches_reference():
    """the structured 64^5 twin of test_gpu_fullgolden.py (its input builder), streamed in 64 MiB chunks from pageable
    memory: the reference's ranks and error within 1e-5; the error from the norm alone agrees."""
    from tntorch_b200 import ops

    g = np.load(os.path.join(GOLD, "full.npz"))
    name = "twin64x5_r32_f32"
    spec = cases.FULL_TTSVD_CASES[name]
    X = torch.from_numpy(cases.make_dense_big(spec))
    cores, info = ops.ttsvd_stream(X, rmax=spec["ranks_tt"], chunk_bytes=64 << 20, return_info=True)
    assert info["chunks"] == 64 and info["passes"] == 2, info
    assert [1] + [int(c.shape[2]) for c in cores] == list(g[f"{name}/eig/ranks"])
    Xd = X.cuda()
    err = ops.tt_relative_error(Xd, cores)
    assert abs(err - float(g[f"{name}/eig/relerr"])) <= 1e-5, err
    assert abs(ops.tt_relative_error_from_norm(info["norm"], cores) - err) <= _from_norm_tol(err)
