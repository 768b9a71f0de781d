"""H100: tn.tt_multiply / ops.tt_multiply (tnb_tt_multiply) against the reference's goldens and an fp64 oracle, path by
path: every branch of the step chooser (asserted by launch count), exactness on small integers, zero, 3-D,
non-contiguous and misaligned inputs, canaries, two streams, no host synchronisation, the error behaviour of the
reference, gradients through the einsum chain, C-ABI refusals, an intermediate past 2^31 elements and the benchmark's
rank-16 shape."""
import ctypes
import os
import threading

import numpy as np
import pytest
import torch

import ttm_model as tm

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = torch.float32

# name -> (input dims, output dims, inner ranks, batch, dtype); the paths each step takes follow from ttm_model
CASES = {
    "d1_prime_b127": ([13], [11], [], 127, F32),
    "d1_b1_f64": ([7], [5], [], 1, torch.float64),
    "d2_r16_tc_b4097": ([8, 16], [64, 4], [16], 4097, F32),
    "d2_r16_n_odd": ([8, 16], [64, 3], [16], 4097, F32),
    "d2_r16_few_rows_b3": ([4, 4], [4, 4], [16], 3, F32),
    "d3_r16_tc": ([8, 8, 8], [8, 8, 8], [16, 16], 4097, F32),
    "d3_r4_r12_tc": ([8, 8, 8], [8, 8, 8], [4, 12], 4097, F32),
    "d3_r16_r25_two_col_tiles": ([8, 8, 8], [8, 8, 8], [16, 25], 1024, F32),
    "d3_r36_two_r_chunks": ([4, 8, 8], [8, 8, 4], [36, 36], 127, F32),
    "d3_r64_small_last": ([4, 8, 8], [8, 8, 4], [64, 64], 127, F32),
    "d3_r256_tc": ([4, 2, 8], [8, 2, 3], [256, 2], 4097, F32),
    "d3_r260_past_limit": ([4, 2, 8], [8, 2, 3], [260, 2], 4097, F32),
    "d3_r7": ([5, 7, 3], [3, 7, 5], [7, 7], 127, F32),
    "d3_r16_f64": ([8, 8, 8], [8, 8, 8], [16, 16], 127, torch.float64),
    "d4_r16_b127": ([8, 8, 8, 8], [8, 8, 8, 8], [16, 16, 16], 127, F32),
    "d4_unit_modes_b1": ([1, 3, 4, 1], [2, 1, 5, 3], [2, 3, 1], 1, F32),
    "d5_r8_b3": ([4] * 5, [4] * 5, [8] * 4, 3, F32),
    "d6_primes_ones_b127": ([2, 3, 1, 5, 2, 2], [3, 1, 2, 2, 5, 1], [3, 7, 5, 4, 2], 127, F32),
    "d6_primes_ones_f64": ([2, 3, 1, 5, 2, 2], [3, 1, 2, 2, 5, 1], [3, 7, 5, 4, 2], 127, torch.float64),
    "d3_r1": ([8, 8, 8], [8, 8, 8], [1, 1], 4097, F32),
}
# the C-ABI case whose Y is offset by one element: its last step leaves the tensor-core path for that reason alone
MISALIGNED_Y_CASE = "d3_r16_tc"


def case_paths(name, y_aligned=True):
    idims, odims, inner, nb, dtype = CASES[name]
    return tm.paths(dtype == F32, idims, odims, [1] + inner + [1], nb, y_aligned)


def _cores(idims, odims, inner, dtype, seed, integer=False):
    g = torch.Generator().manual_seed(seed)
    r = [1] + inner + [1]
    out = []
    for k in range(len(idims)):
        shape = (r[k], idims[k], odims[k], r[k + 1])
        c = torch.randint(-1, 2, shape, generator=g).double() if integer else torch.randn(shape, generator=g, dtype=torch.float64)
        out.append((c if integer else c / np.sqrt(r[k] * idims[k])).to(dtype))
    return out


def _x(nb, I, dtype, seed, integer=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-2, 3, (nb, I), generator=g).double() if integer else torch.randn(nb, I, generator=g, dtype=torch.float64)
    return x.to(dtype)


def _dense(cores):
    """M (I x O) in fp64 on the host, from cores [r, i, o, r']."""
    M = np.ones((1, 1, 1))
    for c in cores:
        c = c.detach().cpu().double().numpy()
        M = np.einsum("abr,rios->aibos", M, c).reshape(M.shape[0] * c.shape[1], M.shape[1] * c.shape[2], c.shape[3])
    return M[:, :, 0]


def _ttm(cores, idims, odims):
    import tntorch_b200 as tnb

    return tnb.TTMatrix(list(cores), ranks=[c.shape[-1] for c in cores[:-1]], input_dims=idims, output_dims=odims)


def _floor(d):
    """The error of d fp32 roundings: a chain stores each of its d step results in fp32 once, whatever it computes in."""
    return d * 2.0 ** -24


def _errors(Y, Y64, bound):
    """normwise relative error and the largest |Y - Y64| / (|X| |M|)"""
    D = np.abs(np.asarray(Y, dtype=np.float64) - Y64)
    return np.linalg.norm(D) / np.linalg.norm(Y64), float(np.max(D / np.maximum(bound, 1e-300)))


def _ref_chain_cpu(cores, X, idims, odims):
    from tntorch_b200.callers import _tt_multiply_einsum

    return _tt_multiply_einsum(_ttm([c.cpu() for c in cores], idims, odims), X.cpu()).numpy()


def test_path_coverage():
    """Every branch of ttm_step_path is taken by some step of the cases below (CPU, no device needed)."""
    seen = {p for n in CASES for p in case_paths(n)} | set(case_paths(MISALIGNED_Y_CASE, y_aligned=False))
    assert seen == set(tm.BRANCHES), {tm.BRANCHES[b] for b in set(tm.BRANCHES) - seen}
    assert {len(c[0]) for c in CASES.values()} >= {1, 2, 3, 4, 5, 6}
    assert {1, 7, 16, 64, 256, 260} <= {r for c in CASES.values() for r in c[2]}
    assert {1, 3, 127, 4097} <= {c[3] for c in CASES.values()}
    assert case_paths(MISALIGNED_Y_CASE)[-1] == tm.TC and case_paths(MISALIGNED_Y_CASE, False)[-1] == tm.OUT_ALIGN


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted({k.split("/")[0] for k in np.load(os.path.join(REPO, "tests", "golden", "tt_multiply.npz")).files}))
def test_golden(name):
    import tntorch_b200 as tnb

    G = np.load(os.path.join(REPO, "tests", "golden", "tt_multiply.npz"))
    cores = [torch.from_numpy(G[f"{name}/core{k}"]).cuda() for k in range(int(G[f"{name}/d"]))]
    idims, odims = G[f"{name}/input_dims"].tolist(), G[f"{name}/output_dims"].tolist()
    X, Yref = torch.from_numpy(G[f"{name}/X"]).cuda(), G[f"{name}/Y"]
    Y = tnb.tt_multiply(_ttm(cores, idims, odims), X)
    assert Y.dtype == cores[0].dtype and Y.device == X.device and tuple(Y.shape) == Yref.shape
    Y = Y.cpu().numpy()
    if Yref.dtype == np.float64:
        assert np.linalg.norm(Y - Yref) <= 1e-12 * np.linalg.norm(Yref)
    else:
        c64 = [c.double() for c in cores]
        Y64 = X.double().cpu().numpy().reshape(Yref.shape[0], -1) @ _dense(c64)
        bound = np.abs(X.double().cpu().numpy().reshape(Yref.shape[0], -1)) @ _dense([c.abs() for c in c64])
        ours, ref = _errors(Y, Y64, bound), _errors(Yref, Y64, bound)
        for o, r in zip(ours, ref):
            assert o <= max(2 * r, _floor(len(cores))), (ours, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_against_fp64(name):
    from tntorch_b200 import ops

    idims, odims, inner, nb, dtype = CASES[name]
    cores = [c.cuda() for c in _cores(idims, odims, inner, dtype, seed=len(name))]
    X = _x(nb, int(np.prod(idims)), dtype, seed=7).cuda()
    n0 = ops.launch_count()
    Y = ops.tt_multiply(cores, X)
    assert ops.launch_count() - n0 == tm.launches(dtype == F32, idims, odims, [1] + inner + [1], nb), case_paths(name)
    M64 = _dense(cores)
    X64 = X.double().cpu().numpy()
    Y64 = X64 @ M64
    if dtype == torch.float64:
        assert np.linalg.norm(Y.cpu().numpy() - Y64) <= 1e-12 * np.linalg.norm(Y64)
        return
    bound = np.abs(X64) @ _dense([c.abs() for c in cores])
    ours = _errors(Y.cpu().numpy(), Y64, bound)
    ref = _errors(_ref_chain_cpu(cores, X, idims, odims), Y64, bound)
    for o, r in zip(ours, ref):
        assert o <= max(2 * r, _floor(len(idims))), (name, ours, ref, case_paths(name))


@pytest.mark.gpu
def test_small_integers_are_exact():
    from tntorch_b200 import ops

    idims, odims, inner, nb, _ = CASES["d3_r16_tc"]
    assert case_paths("d3_r16_tc")[1:] == [tm.TC, tm.TC]
    c32 = [c.cuda() for c in _cores(idims, odims, inner, F32, seed=3, integer=True)]
    X = _x(nb, 512, F32, seed=4, integer=True).cuda()
    Y32 = ops.tt_multiply(c32, X)
    Y64 = ops.tt_multiply([c.double() for c in c32], X.double())
    assert torch.equal(Y32.double(), Y64)


@pytest.mark.gpu
def test_zero_3d_noncontiguous_and_misaligned_inputs():
    import tntorch_b200 as tnb

    idims, odims, inner, nb, _ = CASES["d3_r16_tc"]
    cores = [c.cuda() for c in _cores(idims, odims, inner, F32, seed=5)]
    ttm = _ttm(cores, idims, odims)
    assert torch.count_nonzero(tnb.tt_multiply(ttm, torch.zeros(nb, 512, device="cuda"))) == 0
    X = _x(nb, 512, F32, seed=6).cuda()
    want = tnb.tt_multiply(ttm, X)
    assert torch.equal(tnb.tt_multiply(ttm, X.reshape(nb, 8, 64)), want)  # 3-D
    Xt = X.t().contiguous().t()
    assert not Xt.is_contiguous() and torch.equal(tnb.tt_multiply(ttm, Xt), want)
    buf = torch.empty(nb * 512 + 1, device="cuda")
    Xo = buf[1:].view(nb, 512)
    Xo.copy_(X)
    assert Xo.data_ptr() % 16 != 0 and torch.equal(tnb.tt_multiply(ttm, Xo), want)


def _abi_call(cores, idims, odims, ranks, X, nb, Y, ws, wsb, stream=None):
    from tntorch_b200 import _lib, ops

    code = ops._dtype_code(cores[0])
    ptrs = (ctypes.c_void_p * len(cores))(*[c.data_ptr() for c in cores])
    return _lib.lib().tnb_tt_multiply(code, ptrs, len(cores), _lib.i64(idims), _lib.i64(odims), _lib.i32(ranks),
                                      ctypes.c_void_p(X.data_ptr()), nb, ctypes.c_void_p(Y.data_ptr()),
                                      ctypes.c_void_p(ws.data_ptr()), wsb,
                                      ctypes.c_void_p(stream if stream is not None else torch.cuda.current_stream().cuda_stream))


@pytest.mark.gpu
def test_canaries_and_misaligned_y():
    from tntorch_b200 import _lib, ops

    name = MISALIGNED_Y_CASE
    idims, odims, inner, nb, _ = CASES[name]
    ranks = [1] + inner + [1]
    cores = [c.cuda() for c in _cores(idims, odims, inner, F32, seed=8)]
    X = _x(nb, 512, F32, seed=9).cuda()
    want = ops.tt_multiply(cores, X)
    wsb = _lib.lib().tnb_tt_multiply_workspace_bytes(_lib.TNB_F32, 3, _lib.i64(idims), _lib.i64(odims), _lib.i32(ranks), nb)
    assert wsb == tm.workspace_bytes(True, idims, odims, ranks, nb)
    pad = 4096
    wbuf = torch.full((wsb + 2 * pad,), 0xA5, dtype=torch.uint8, device="cuda")
    O = 512
    for off in (4, 1):  # 16-byte aligned Y, then Y offset by one element (its last step on the generic tiles)
        ybuf = torch.full((nb * O + 2 * 1024,), 12345.0, device="cuda")
        Y = ybuf[1024 - 4 + off: 1024 - 4 + off + nb * O].view(nb, O)
        n0 = ops.launch_count()
        assert _abi_call(cores, idims, odims, ranks, X, nb, Y, wbuf[pad:pad + wsb], wsb) == 0
        assert ops.launch_count() - n0 == tm.launches(True, idims, odims, ranks, nb, y_aligned=(off == 4))
        torch.cuda.synchronize()
        assert (wbuf[:pad] == 0xA5).all() and (wbuf[pad + wsb:] == 0xA5).all()
        start = 1024 - 4 + off
        assert (ybuf[:start] == 12345.0).all() and (ybuf[start + nb * O:] == 12345.0).all()
        assert torch.allclose(Y, want, rtol=1e-5, atol=1e-5 * want.abs().max().item())


@pytest.mark.gpu
def test_abi_refusals_leave_y_untouched():
    from tntorch_b200 import _lib

    idims, odims, inner, nb, _ = CASES["d3_r16_tc"]
    ranks = [1] + inner + [1]
    cores = [c.cuda() for c in _cores(idims, odims, inner, F32, seed=10)]
    X = _x(nb, 512, F32, seed=11).cuda()
    Y = torch.full((nb, 512), 7.0, device="cuda")
    wsb = _lib.lib().tnb_tt_multiply_workspace_bytes(_lib.TNB_F32, 3, _lib.i64(idims), _lib.i64(odims), _lib.i32(ranks), nb)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    assert _abi_call(cores, idims, odims, ranks, X, nb, Y, ws, wsb - 1) == _lib.ERR_WORKSPACE
    assert _abi_call(cores, idims, odims, [2] + inner + [1], X, nb, Y, ws, wsb) == _lib.ERR_INVALID
    assert _abi_call(cores, [8, 0, 8], odims, ranks, X, nb, Y, ws, wsb) == _lib.ERR_INVALID
    assert _abi_call(cores, idims, odims, ranks, X, 0, Y, ws, wsb) == _lib.ERR_INVALID
    assert _abi_call(cores, idims, odims, ranks, X, 1 << 31, Y, ws, wsb) == _lib.ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert (Y == 7.0).all()


@pytest.mark.gpu
def test_two_threads_two_streams():
    from tntorch_b200 import ops

    idims, odims, inner, nb, _ = CASES["d3_r16_tc"]
    sets = [([c.cuda() for c in _cores(idims, odims, inner, F32, seed=20 + i)], _x(nb, 512, F32, seed=30 + i).cuda())
            for i in range(2)]
    want = [ops.tt_multiply(c, x) for c, x in sets]
    got = [None, None]

    def run(i):
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            for _ in range(3):
                got[i] = ops.tt_multiply(*sets[i])
        s.synchronize()

    th = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    [t.start() for t in th]
    [t.join() for t in th]
    for i in range(2):
        assert torch.equal(got[i], want[i])


@pytest.mark.gpu
def test_no_host_synchronisation():
    from tntorch_b200 import ops

    idims, odims, inner, nb, _ = CASES["d3_r16_tc"]
    cores = [c.cuda() for c in _cores(idims, odims, inner, F32, seed=12)]
    X = _x(nb, 512, F32, seed=13).cuda()
    ops.tt_multiply(cores, X)  # load the library and set kernel attributes first
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ops.tt_multiply(cores, X)
    finally:
        torch.cuda.set_sync_debug_mode("default")


@pytest.mark.gpu
def test_errors_like_the_reference():
    import tntorch_b200 as tnb

    idims, odims, inner = [11, 3], [23, 2], [6]
    cores = [c.cuda() for c in _cores(idims, odims, inner, torch.float64, seed=14)]
    ttm = _ttm(cores, idims, odims)
    with pytest.raises(AssertionError):
        tnb.tt_multiply(ttm, torch.zeros(33, dtype=torch.float64, device="cuda"))
    with pytest.raises(RuntimeError):
        tnb.tt_multiply(ttm, torch.zeros(5, 7, dtype=torch.float64, device="cuda"))  # 35 does not divide by 33
    with pytest.raises(RuntimeError):
        tnb.tt_multiply(ttm, torch.zeros(4, 33, dtype=torch.float32, device="cuda"))
    with pytest.raises(RuntimeError):
        tnb.tt_multiply(ttm, torch.zeros(4, 33, dtype=torch.float64))
    batched = tnb.TTMatrix([c[None].expand(2, *c.shape) for c in cores], ranks=inner, input_dims=idims, output_dims=odims)
    with pytest.raises(NotImplementedError):
        tnb.tt_multiply(batched, torch.zeros(4, 33, dtype=torch.float64, device="cuda"))
    from tntorch_b200 import ops

    with pytest.raises(NotImplementedError):
        ops.tt_multiply(batched.cores, torch.zeros(4, 33, dtype=torch.float64, device="cuda"))


@pytest.mark.gpu
def test_gradients_through_the_einsum_chain():
    import tntorch_b200 as tnb

    idims, odims, inner = [4, 3, 5], [2, 3, 2], [3, 4]
    base = [c.cuda() for c in _cores(idims, odims, inner, torch.float64, seed=15)]
    X0 = _x(6, 60, torch.float64, seed=16).cuda()
    grads = []
    for use_lib in (True, False):
        cores = [c.clone().requires_grad_() for c in base]
        X = X0.clone().requires_grad_()
        if use_lib:
            Y = tnb.tt_multiply(_ttm(cores, idims, odims), X)
        else:  # the reference's chain, written out
            r = X.reshape(6, -1).T.reshape(idims[0], -1)
            r = torch.einsum("id,lior->ldor", r, cores[0])
            for k in range(1, 3):
                r = torch.einsum("idr,riob->dob", r.reshape(idims[k], -1, cores[k].shape[0]), cores[k])
            Y = r.reshape(6, -1)
        (Y * torch.arange(Y.numel(), device="cuda", dtype=Y.dtype).reshape(Y.shape)).sum().backward()
        grads.append([X.grad] + [c.grad for c in cores])
    for a, b in zip(*grads):
        assert torch.allclose(a, b, rtol=1e-12, atol=0)
    with torch.no_grad():
        assert torch.allclose(tnb.tt_multiply(_ttm(base, idims, odims), X0), X0 @ torch.from_numpy(_dense(base)).cuda())


@pytest.mark.gpu
def test_full_rank_ttmatrix_reproduces_x_times_m():
    import tntorch_b200 as tnb

    g = torch.Generator().manual_seed(17)
    M = torch.randn(24, 20, generator=g, dtype=torch.float64).cuda()
    ttm = tnb.TTMatrix(M, ranks=[10, 8], input_dims=[2, 3, 4], output_dims=[5, 2, 2])
    X = torch.randn(9, 24, generator=g, dtype=torch.float64).cuda()
    Y = tnb.tt_multiply(ttm, X)
    assert torch.linalg.norm(Y - X @ M) <= 1e-10 * torch.linalg.norm(X @ M)


def _sampled_rows_check(idims, odims, inner, nb, seed):
    from tntorch_b200 import ops

    cores = [c.cuda() for c in _cores(idims, odims, inner, F32, seed=seed)]
    I = int(np.prod(idims))
    X = torch.randn(nb, I, generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda")
    n0 = ops.launch_count()
    Y = ops.tt_multiply(cores, X)
    assert ops.launch_count() - n0 == tm.launches(True, idims, odims, [1] + inner + [1], nb)
    rows = torch.linspace(0, nb - 1, 64).long()
    Xs = X[rows].double().cpu().numpy()
    Y64 = Xs @ _dense(cores)
    bound = np.abs(Xs) @ _dense([c.abs() for c in cores])
    ours = _errors(Y[rows].cpu().numpy(), Y64, bound)
    ref = _errors(_ref_chain_cpu(cores, X[rows], idims, odims), Y64, bound)
    for o, r in zip(ours, ref):
        assert o <= max(2 * r, _floor(len(idims))), (ours, ref)


@pytest.mark.gpu
def test_intermediate_past_2_31_elements():
    idims, odims, inner, nb = [8] * 4, [8] * 4, [32] * 3, 16400
    st = tm.steps(idims, odims, [1] + inner + [1])
    assert max(nb * R * N for R, _, _, N in st[:-1]) > 2 ** 31
    _sampled_rows_check(idims, odims, inner, nb, seed=18)


@pytest.mark.gpu
def test_benchmark_rank16_shape():
    idims, odims, inner, nb = [8] * 4, [8] * 4, [16] * 3, 8192
    assert tm.paths(True, idims, odims, [1] + inner + [1], nb) == [tm.RANK_ALIGN, tm.TC, tm.TC, tm.TC]
    _sampled_rows_check(idims, odims, inner, nb, seed=19)
