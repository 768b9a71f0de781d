"""GPU: ops.tt_hadamard_round (tnb_tt_hadamard_round) against the reference's own results (tests/golden/hadamard_round.npz),
every path in both dtypes against the fp64 model and oracle, against today's Kronecker + tt_round path where that runs,
the routing of tn.reduce and tn.hadamard_sum, config 3, and the call contract."""
import json
import math
import operator
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import tthr_model as hm
import tntorch_b200 as tn
from tntorch_b200 import callers, ops

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hadamard_round.npz")
# the bounds tests/test_gpu_round_paths.py holds tnb_tt_round to
TOL = {
    torch.float64: dict(relerr=1e-8, orth=1e-10),
    torch.float32: dict(relerr=1e-5, orth=1e-5),
}


def _tt(seed, shape, ranks, dtype, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    r = [1] + list(ranks) + [1]
    return [(scale * torch.randn(r[k], shape[k], r[k + 1], generator=g, dtype=torch.float64)).to(dtype).cuda()
            for k in range(len(shape))]


def _np(cores):
    return [c.detach().cpu().double().numpy() for c in cores]


def _ranks(cores):
    return [1] + [int(c.shape[2]) for c in cores]


def _relerr_to_product(a, b, cores):
    """||a*b - cores|| / ||a*b|| from three TT dots in fp64 (hadamard products formed on the host for small cases)."""
    exact = hm.full(hm.kronecker(_np(a), _np(b)))
    return float(np.linalg.norm(hm.full(_np(cores)) - exact) / np.linalg.norm(exact))


def _orth(cores, tol):
    for c in cores[1:]:
        M = c.double().reshape(c.shape[0], -1)
        assert torch.allclose(M @ M.T, torch.eye(M.shape[0], dtype=torch.float64, device=M.device), atol=tol)


def _kernels(fn):
    """(tensor-core, CUDA-core) launches of the tthr GEMM kernels `fn` makes.  Every call launches at least one (core 0),
    so a trace without any came back empty: it is taken again, and an empty one is never accepted."""
    from torch.profiler import ProfilerActivity, profile

    fn()  # first-call setup out of the trace
    torch.cuda.synchronize()
    counts = (0, 0)
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        counts = (sum("tthr_gemm_tc_kernel" in n for n in names), sum("tthr_gemm_generic_kernel" in n for n in names))
        if sum(counts) > 0:
            break
    assert sum(counts) > 0, "the profiler recorded no tthr_ kernel"
    return counts


# ------------------------------------------------------------------ the reference's own results
def test_reference_goldens():
    g = np.load(GOLDEN)
    names = sorted({k.split("/")[0] for k in g.files if k.endswith("/relerr") and f"{k.split('/')[0]}/a0" in g.files})
    assert len(names) >= 8
    for name in names:
        N = int(g[f"{name}/N"])
        a = [torch.as_tensor(g[f"{name}/a{k}"]).cuda() for k in range(N)]
        # the reference's CP conversion builds float32 cores whatever the factors' dtype: both operands in a's dtype
        b = [torch.as_tensor(g[f"{name}/b{k}"]).to(a[0].dtype).cuda() for k in range(N)]
        eps, rmax = float(g[f"{name}/eps"]), int(g[f"{name}/rmax"])
        cores = ops.tt_hadamard_round(a, b, eps=eps, rmax=rmax if rmax > 0 else None)
        assert _ranks(cores) == list(g[f"{name}/ranks"]), name
        assert cores[0].dtype == a[0].dtype
        if name.startswith("zero"):
            assert all(not torch.any(c) for c in cores)
            continue
        err = _relerr_to_product(a, b, cores)
        assert abs(err - float(g[f"{name}/relerr"])) < 1e-5, (name, err)


def test_reference_goldens_reduce_and_hadamard_sum():
    g = np.load(GOLDEN)
    for tag in ("f64", "f32"):
        ts = [tn.Tensor([torch.as_tensor(g[f"reduce_{tag}/t{i}_{k}"]).cuda() for k in range(5)]) for i in range(4)]
        r = tn.reduce(ts, operator.mul, eps=1e-3)
        full = ts[0].torch().double() * ts[1].torch().double() * ts[2].torch().double() * ts[3].torch().double()
        err = float(torch.norm(full - r.torch().double()) / torch.norm(full))
        assert abs(err - float(g[f"reduce_{tag}/relerr"])) < 1e-5
        assert [int(x) for x in r.ranks_tt] == list(g[f"reduce_{tag}/ranks"]) or tag == "f32"
    ts = [tn.Tensor([torch.as_tensor(g[f"hsum_f32/t{i}_{k}"]).cuda() for k in range(4)]) for i in range(3)]
    exact = float(g["hsum_f32/exact"])
    ref_gap = abs(float(g["hsum_f32/svd"]) - exact)
    assert abs(tn.hadamard_sum(ts, algorithm="svd", eps=1e-6) - exact) <= max(2 * ref_gap, 1e-4 * abs(exact))


# ------------------------------------------------------------------ every path, both dtypes, against the fp64 model
PATH_CASES = [
    # name, shape, ranks a, ranks b, eps, rmax, tensor-core kernel expected (with the tensor cores allowed)
    ("tc_modes", [6] * 5, [16, 24, 24, 16], [16, 16, 20, 16], 1e-6, 40, True),
    ("generic_modes", [5] * 5, [3, 5, 5, 3], [2, 4, 4, 2], 1e-10, None, False),
    ("r576_eps", [4] * 6, [24] * 5, [24] * 5, 1e-2, None, True),
    ("wide_bond_chfsi", [40, 40, 40], [20, 20], [20, 20], 0.0, 30, True),
    ("n2", [7, 9], [5], [4], 1e-10, None, False),
    ("n1", [11], [], [], 1e-14, None, False),
]


def _path_args(case, use_tc, dtype):
    _, shape, ra, rb, eps, rmax, tc_expected = next(c for c in PATH_CASES if c[0] == case)
    a, b = _tt(1, shape, ra, dtype), _tt(2, shape, rb, dtype)
    return shape, a, b, eps, rmax, tc_expected


def trace_path_cases():
    """{"case/use_tc/dtype": [tensor-core launches, CUDA-core launches]} of every path case, and "syncs": [N, host
    synchronisations] of one call (sync_count)."""
    out = {}
    for case in [c[0] for c in PATH_CASES]:
        for use_tc in (True, False):
            for dtype in (torch.float64, torch.float32):
                shape, a, b, eps, rmax, _ = _path_args(case, use_tc, dtype)
                out[f"{case}/{use_tc}/{dtype}"] = list(_kernels(
                    lambda: ops.tt_hadamard_round(a, b, eps=eps, rmax=rmax, use_tensorcore=use_tc)))
    out["syncs"] = list(sync_count())
    return out


@pytest.fixture(scope="module")
def path_kernels():
    """The kernels of every path case, traced in a fresh process: late in a long process that has profiled before, the
    activity trace has come back without some of the kernels a call launched."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here, os.environ.get("PYTHONPATH", "")]))
    code = "import json, test_gpu_tt_hadamard_round as t; print('TRACE ' + json.dumps(t.trace_path_cases()))"
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=os.path.dirname(here),
                       timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    line = [x for x in r.stdout.splitlines() if x.startswith("TRACE ")][-1]
    return json.loads(line[len("TRACE "):])


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("use_tc", [True, False])
@pytest.mark.parametrize("case", [c[0] for c in PATH_CASES])
def test_paths_against_model(case, use_tc, dtype, path_kernels):
    shape, a, b, eps, rmax, tc_expected = _path_args(case, use_tc, dtype)
    N = len(shape)
    rm = None if rmax is None else [rmax] * (N - 1)
    cores, info = ops.tt_hadamard_round(a, b, eps=eps, rmax=rmax, return_info=True, use_tensorcore=use_tc)
    tc_launches, gen_launches = path_kernels[f"{case}/{use_tc}/{dtype}"]
    if not use_tc:
        assert tc_launches == 0 and gen_launches > 0
    elif tc_expected:
        assert tc_launches > 0
    # launches: four per chunk of each mode of the recurrence, two for core 0 and at most five GEMMs per bond
    assert tc_launches + gen_launches <= 4 * sum(shape[:-1]) + 2 + 5 * (N - 1)
    mcores, mranks, mnorm, mdisc = hm.hadamard_round(_np(a), _np(b), eps=eps, rmax=rm)
    assert _ranks(cores) == mranks
    err = _relerr_to_product(a, b, cores)
    exact = hm.full(hm.kronecker(_np(a), _np(b)))
    merr = float(np.linalg.norm(hm.full(mcores) - exact) / np.linalg.norm(exact))
    assert abs(err - merr) <= TOL[dtype]["relerr"] + 1e-6 * merr
    _orth(cores, TOL[dtype]["orth"])
    assert info["norm_sq"] == pytest.approx(mnorm, rel=1e-10)
    if dtype == torch.float64 and err > 1e-6:
        assert math.sqrt(info["discarded_sq"] / info["norm_sq"]) == pytest.approx(err, rel=1e-6)


# ------------------------------------------------------------------ against today's Kronecker + tt_round path
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_same_as_kronecker_path_where_it_runs(dtype):
    shape = [8] * 5
    a, b = _tt(3, shape, [4, 8, 8, 4], dtype), _tt(4, shape, [4, 8, 8, 4], dtype)
    for eps, rmax in ((1e-3, None), (0.0, 12)):
        fused = ops.tt_hadamard_round(a, b, eps=eps, rmax=rmax)
        old = ops.tt_round(ops.tt_hadamard(a, b), eps=eps, rmax=rmax)
        assert _ranks(fused) == _ranks(old)
        e_f, e_o = _relerr_to_product(a, b, fused), _relerr_to_product(a, b, old)
        assert abs(e_f - e_o) <= TOL[dtype]["relerr"] + 1e-6 * e_o


def test_reduce_and_hadamard_sum_unchanged_where_kronecker_runs():
    shape = [8] * 5
    ts = [tn.Tensor(_tt(10 + k, shape, [4] * 4, torch.float64)) for k in range(4)]
    assert not ops.hadamard_round_instead_of_kronecker(shape, [1] + [4] * 4 + [1], [1] + [4] * 4 + [1], 8,
                                                       torch.cuda.mem_get_info()[0])

    def old_node(x, y):
        out = x * y
        out.round(eps=1e-4)
        return out

    n0 = ops.launch_count()
    r = tn.reduce(ts, operator.mul, eps=1e-4)
    n_new = ops.launch_count() - n0
    n0 = ops.launch_count()
    ref = old_node(old_node(ts[0], ts[1]), old_node(ts[2], ts[3]))
    n_old = ops.launch_count() - n0
    assert n_new == n_old
    for c1, c2 in zip(r.cores, ref.cores):
        assert torch.equal(c1, c2)
    cs = [t._tt_cores() for t in ts[:3]]
    step = 1e-6 / math.sqrt(2)
    P = ops.tt_round(ops.tt_hadamard(ops.tt_round(ops.tt_hadamard(cs[0], cs[1]), eps=step), cs[2]), eps=step)
    assert tn.hadamard_sum(ts[:3], algorithm="svd", eps=1e-6) == float(callers._sum_all(P))


def test_kronecker_path_still_refuses_above_256():
    shape = [4] * 5
    a, b = _tt(5, shape, [17] * 4, torch.float64), _tt(6, shape, [17] * 4, torch.float64)
    with pytest.raises(NotImplementedError):
        ops.tt_round(ops.tt_hadamard(a, b))
    assert ops.hadamard_round_instead_of_kronecker(shape, _ranks(a), _ranks(b), 8, 80 << 30)
    cores = ops.tt_hadamard_round(a, b, eps=1e-6)
    assert _relerr_to_product(a, b, cores) < 1e-6
    # tn.reduce and tn.hadamard_sum take the fused call there
    ta, tb = tn.Tensor(a), tn.Tensor(b)
    r = tn.reduce([ta, tb], operator.mul, eps=1e-6)
    assert _relerr_to_product(a, b, r._tt_cores()) < 1e-6
    exact = tn.hadamard_sum([ta, tb], algorithm="exact")
    assert tn.hadamard_sum([ta, tb], algorithm="svd", eps=1e-10) == pytest.approx(exact, rel=1e-8)


# ------------------------------------------------------------------ config 3 (128^10, rank 64, fp64)
def _ones_at_rank(shape, r, seed):
    """The all-ones tensor written at rank r with random invertible gauges G_k: core_k[:, i, :] = G_k^-1 J G_{k+1},
    J = 1 1^T / r (a projector), first core 1^T J G_1 / sqrt(r), last G_{N-1}^-1 J 1 / sqrt(r)."""
    g = torch.Generator().manual_seed(seed)
    N = len(shape)
    J = torch.full((r, r), 1.0 / r, dtype=torch.float64)
    G = [torch.eye(r, dtype=torch.float64) + 0.1 * torch.randn(r, r, generator=g, dtype=torch.float64) / math.sqrt(r)
         for _ in range(N + 1)]
    one = torch.ones(r, dtype=torch.float64) / math.sqrt(r)
    cores = []
    for k in range(N):
        if k == 0:
            M = (one @ J @ G[1])[None, :]
        elif k == N - 1:
            M = (torch.linalg.solve(G[k], J @ one))[:, None]
        else:
            M = torch.linalg.solve(G[k], J @ G[k + 1])
        cores.append(M[:, None, :].expand(M.shape[0], shape[k], M.shape[1]).contiguous().cuda())
    return cores


def test_config3_times_ones_is_exact():
    shape = [128] * 10
    A = _tt(20, shape, [64] * 9, torch.float64)
    B = _ones_at_rank(shape, 64, 21)
    ta = tn.Tensor(A)
    # eps = 1e-9 sits below the Gram's noise floor at a bond Gram of 8192 (Gram-class rounding, DESIGN §6): with the cap at
    # A's rank the rank rule returns it; eps = 1e-5 finds it without a cap
    for eps, rmax in ((1e-9, 64), (1e-5, None)):
        cores = ops.tt_hadamard_round(A, B, eps=eps, rmax=rmax)
        assert _ranks(cores) == _ranks(A)
        assert float(tn.dist(tn.Tensor(cores), ta) / tn.norm(ta)) <= 1e-7


def test_config3_square_rmax16_energies():
    shape = [128] * 10
    t = _tt(22, shape, [64] * 9, torch.float64, scale=1 / 8)
    torch.cuda.reset_peak_memory_stats()
    cores, info = ops.tt_hadamard_round(t, t, eps=1e-14, rmax=16, return_info=True)
    assert torch.cuda.max_memory_allocated() < 80e9
    assert _ranks(cores) == [1] + [16] * 9 + [1]
    tt_, R = tn.Tensor(t), tn.Tensor(cores)
    cc = info["norm_sq"]
    cr = tn.hadamard_sum([tt_, tt_, R], algorithm="exact")
    rr = float(ops.tt_dot(cores, cores))
    err2 = cc - 2 * cr + rr
    assert err2 / cc == pytest.approx(info["discarded_sq"] / cc, rel=1e-6, abs=1e-10)


def test_config3_reduce_four_rmax16():
    shape = [128] * 10
    ts = [tn.Tensor(_tt(30 + k, shape, [64] * 9, torch.float64, scale=1 / 8)) for k in range(4)]
    r = tn.reduce(ts, operator.mul, rmax=16)
    assert max(int(x) for x in r.ranks_tt) <= 16


# ------------------------------------------------------------------ the call contract
def test_bitwise_reproducible_and_two_streams():
    shape = [6] * 5
    a, b = _tt(40, shape, [16, 24, 24, 16], torch.float64), _tt(41, shape, [16, 20, 20, 16], torch.float64)
    ref = ops.tt_hadamard_round(a, b, eps=1e-8)
    for _ in range(2):
        again = ops.tt_hadamard_round(a, b, eps=1e-8)
        assert all(torch.equal(x, y) for x, y in zip(ref, again))
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s1):
        r1 = ops.tt_hadamard_round(a, b, eps=1e-8)
    with torch.cuda.stream(s2):
        r2 = ops.tt_hadamard_round(b, a, eps=1e-8)
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(ref, r1))
    assert _ranks(r2) == _ranks(ref)


def test_canaries_around_outputs():
    import ctypes as C

    from tntorch_b200 import _lib

    shape = [5, 6, 7]
    a, b = _tt(50, shape, [3, 4], torch.float64), _tt(51, shape, [2, 3], torch.float64)
    L = _lib.lib()
    N = 3
    sh, ra, rb, rm = _lib.i64(shape), _lib.i32(_ranks(a)), _lib.i32(_ranks(b)), _lib.i32([0, 0])
    offs = (C.c_int64 * N)()
    cap = L.tnb_tt_hadamard_round_cores_capacity(N, sh, ra, rb, rm, offs)
    wsb = L.tnb_tt_hadamard_round_workspace_bytes(_lib.TNB_F64, N, sh, ra, rb, rm)
    buf = torch.full((cap + 128,), 7.25, dtype=torch.float64, device="cuda")
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    rk = (C.c_int32 * (N + 1))()
    en = (C.c_double * 2)()
    pa = (C.c_void_p * N)(*[c.data_ptr() for c in a])
    pb = (C.c_void_p * N)(*[c.data_ptr() for c in b])
    rc = L.tnb_tt_hadamard_round(_lib.TNB_F64, pa, pb, N, sh, ra, rb, rm, 1e-12, 0, C.c_void_p(ws.data_ptr()), wsb,
                                 C.c_void_p(buf[64:].data_ptr()), cap, rk, en, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    torch.cuda.synchronize()
    assert torch.all(buf[:64] == 7.25) and torch.all(buf[64 + cap:] == 7.25)
    # a short workspace and mixed dtypes are refused before anything is written
    n0 = ops.launch_count()
    rc = L.tnb_tt_hadamard_round(_lib.TNB_F64, pa, pb, N, sh, ra, rb, rm, 1e-12, 0, C.c_void_p(ws.data_ptr()), 64,
                                 C.c_void_p(buf[64:].data_ptr()), cap, rk, en, None)
    assert rc == _lib.ERR_WORKSPACE and ops.launch_count() == n0
    with pytest.raises(ValueError):
        ops.tt_hadamard_round(a, [c.float() for c in b])
    # the eigen envelope: an rmax above 240 where the bond Gram is wider than 256
    big = [64] * 4
    x, y = _tt(52, big, [16] * 3, torch.float64), _tt(53, big, [16] * 3, torch.float64)
    n0 = ops.launch_count()
    with pytest.raises(NotImplementedError):
        ops.tt_hadamard_round(x, y, rmax=250)
    assert ops.launch_count() == n0


def sync_count():
    """cudaStreamSynchronize calls of one call with rmax at every bond (Jacobi and ChFSI bonds, no adaptive solve).  The
    call always ends in one, so a trace without any came back empty: it is taken again, and an empty one is never
    accepted."""
    from torch.profiler import ProfilerActivity, profile

    shape = [6] * 5
    a, b = _tt(60, shape, [16, 24, 24, 16], torch.float64), _tt(61, shape, [16, 20, 20, 16], torch.float64)
    ops.tt_hadamard_round(a, b, eps=1e-8, rmax=30)
    syncs = 0
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            ops.tt_hadamard_round(a, b, eps=1e-8, rmax=30)
        syncs = sum(1 for e in prof.events() if e.name == "cudaStreamSynchronize")
        if syncs > 0:
            break
    assert syncs > 0, "the profiler recorded no cudaStreamSynchronize"
    return len(shape), syncs


def test_one_synchronisation_per_bond(path_kernels):
    N, syncs = path_kernels["syncs"]
    assert 1 <= syncs <= (N - 1) + 1
