"""-m gpu: entries of tensor trains on the device (tnb_tt_gather through ops.tt_gather / tt_gather_batch and
Tensor.__getitem__).

- the reference's own results on every case of tests/golden/getitem.npz: values, result type, core and factor shapes;
- every branch of ttg_path and ttg_mode_path (restated in tests/ttg_model.py), both dtypes, against the fp64 NumPy chain
  within c K u (the chain in absolute values), the branch seen in the kernels that run and the launches counted;
- bitwise reproducibility, shuffled points giving shuffled outputs, agreement with ops.cross_tt_eval;
- canaries around `out`, refusals that leave `out` alone, two streams on two threads, no host synchronisation;
- config 3 (128^10, rank 64) at P = 2^20, a state past 2^31 elements, rank 256 fp32 on the tensor cores;
- out-of-range keys raise IndexError before anything launches.
"""
import ctypes as C
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

import tntorch_b200 as tn
import ttg_model as tm
from oracle import getitem_cases as gc
from tntorch_b200 import _lib, ops
from test_getitem_oracle import GOLD, case_tensor

pytestmark = pytest.mark.gpu
U = {torch.float64: 2.0 ** -53, torch.float32: 2.0 ** -24}

# name -> (shape, ranks, first, last, P): a case for every branch of ttg_path (ttg_model.PATHS) and of ttg_mode_path
# (ttg_model.BRANCHES)
PATH_CASES = {
    "fused": ([6, 5, 7, 4], [1, 3, 5, 4, 1], 0, 4, 300),
    "fused inner range": ([6, 5, 7, 4], [1, 3, 5, 4, 1], 1, 3, 50),
    "grouped": ([6, 5, 7, 4], [1, 3, 5, 4, 1], 0, 4, 5000),
    "tensor cores": ([6, 5, 7, 4, 3], [1, 16, 24, 20, 32, 1], 0, 5, 6000),
    "tensor cores inner range": ([6, 5, 7, 4, 3], [1, 16, 24, 20, 32, 1], 1, 4, 3000),
    "a rank below 16": ([5, 9, 3], [1, 4, 7, 1], 0, 3, 9000),
    "a rank above 256": ([4, 3, 5], [1, 20, 300, 1], 0, 3, 5000),
    "one mode": ([11], [1, 1], 0, 1, 5000),
}
DTYPES = {"float64": torch.float64, "float32": torch.float32}


def rand_tt(seed, shape, ranks, dtype=torch.float64, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(ranks[k], shape[k], ranks[k + 1], generator=g, dtype=torch.float64) / ranks[k] ** 0.5)
            .to(dtype).to(device) for k in range(len(shape))]


def rand_idx(seed, shape, P, first=0, last=None):
    last = len(shape) if last is None else last
    g = torch.Generator().manual_seed(seed)
    return torch.stack([torch.randint(0, shape[k], (P,), generator=g) for k in range(first, last)], dim=1)


def np_cores(cs):
    return [c.detach().cpu().double().numpy() for c in cs]


def assert_within(got, cores, idx, first, last, dtype, c=4.0):
    """|got - chain| <= c K u |chain|_abs per entry, K the chain depth (ttg_model.depth)."""
    A = np_cores(cores)
    ix = idx.cpu().numpy()
    want = tm.gather(A, ix, first, last)
    absw = tm.gather(A, ix, first, last, absolute=True)
    ranks = [A[0].shape[0]] + [a.shape[2] for a in A]
    K = tm.depth(ranks, first, last) + 1
    err = np.abs(got.detach().cpu().double().numpy() - want)
    lim = c * K * U[dtype] * absw + 1e-300
    assert (err <= lim).all(), float((err / lim).max())


def kernels(fn):
    """Names of the ttg_ kernels `fn` launches, over three calls in one trace."""
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "ttg_" in e.name}
    assert names, "the profiler recorded no ttg_ kernel"
    return sorted(names)


def trace_path_cases():
    """{"name/dtype": kernel names} of one ops.tt_gather per PATH_CASES entry and dtype; run in a process of its own."""
    out = {}
    for name, (shape, ranks, first, last, P) in PATH_CASES.items():
        for dn, dt in DTYPES.items():
            cores = rand_tt(11, shape, ranks, dt)
            idx = rand_idx(12, shape, P, first, last).cuda()
            out[f"{name}/{dn}"] = kernels(lambda: ops.tt_gather(cores, idx, first, last, check=False))
    return out


@pytest.fixture(scope="module")
def path_kernels():
    """The kernels of every path case, traced in a fresh process: late in a long process that has profiled before, the
    activity trace has come back without some of the kernels a call launched."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here, os.environ.get("PYTHONPATH", "")]))
    code = "import json, test_gpu_tt_gather as t; print('TRACE ' + json.dumps(t.trace_path_cases()))"
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=os.path.dirname(here),
                       timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    line = [x for x in r.stdout.splitlines() if x.startswith("TRACE ")][-1]
    return json.loads(line[len("TRACE "):])


# ------------------------------------------------------------------ the reference's goldens
def tensor_for(g, spec, dname):
    cores, Us, batch = case_tensor(g, spec, dname)
    cores = [torch.as_tensor(np.asarray(c)).cuda() for c in cores]
    if Us is not None:
        Us = [None if u is None else torch.as_tensor(np.asarray(u)).cuda() for u in Us]
    return tn.Tensor(cores, Us=Us, batch=batch)


@pytest.mark.parametrize("name,dname", [(n, d) for n in gc.KEYS for d in gc.DTYPES])
def test_golden(name, dname):
    g = np.load(GOLD)
    spec, key = gc.KEYS[name]
    t = tensor_for(g, spec, dname)
    kind = str(g[f"{name}/{dname}/kind"])
    if kind in ("IndexError", "ValueError"):
        with pytest.raises({"IndexError": IndexError, "ValueError": ValueError}[kind]):
            t[key("cuda")]
        return
    r = t[key("cuda")]
    want = g[f"{name}/{dname}/value"]
    tol = 1e-12 if dname == "f64" else 1e-5
    if kind == "scalar":
        assert isinstance(r, torch.Tensor) and r.shape == want.shape
        got = r.cpu().double().numpy()
    else:
        assert isinstance(r, tn.Tensor)
        got = r.torch().cpu().double().numpy()
        if spec != "cp":  # CP cores become TT cores: the values are the reference's, the shapes are not
            shapes = [list(c.shape) + [0] * (4 - c.dim()) for c in r.cores]
            np.testing.assert_array_equal(np.array(shapes), g[f"{name}/{dname}/core_shapes"])
            ushapes = [list(u.shape) + [0] * (3 - u.dim()) if u is not None else [-1, -1, -1] for u in r.Us]
            np.testing.assert_array_equal(np.array(ushapes), g[f"{name}/{dname}/U_shapes"])
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= tol * max(1.0, np.abs(want).max())


# ------------------------------------------------------------------ every branch against the fp64 chain
@pytest.mark.parametrize("dname", list(DTYPES))
@pytest.mark.parametrize("case", list(PATH_CASES))
def test_branch(case, dname, path_kernels):
    dt = DTYPES[dname]
    shape, ranks, first, last, P = PATH_CASES[case]
    cores = rand_tt(11, shape, ranks, dt)
    idx = rand_idx(12, shape, P, first, last).cuda()
    path = tm.path([ranks], first, last, P)
    before = ops.launch_count()
    out = ops.tt_gather(cores, idx, first, last, check=False)
    assert ops.launch_count() - before == tm.launches([ranks], first, last, P)
    assert out.shape == (ranks[first], P, ranks[last]) and out.dtype == dt
    assert_within(out, cores, idx, first, last, dt)
    names = path_kernels[f"{case}/{dname}"]
    want = {tm.PATH_KERNELS[path]}
    if path == tm.GROUPED:
        want |= {tm.MODE_KERNELS[m] for m in tm.mode_paths(ranks, first, last)}
    got = {k for k in ("ttg_fused_kernel", "ttg_init_kernel", "ttg_step_tc_kernel", "ttg_step_generic_kernel")
           if any(k in n for n in names)}
    assert got == want, (names, want)


def test_batch_of_trains_with_their_own_ranks():
    shape = [6, 5, 7, 4]
    trains = [rand_tt(20 + b, shape, [1, 3 + b, 20 - b, 2 + b, 1]) for b in range(3)]
    idx = rand_idx(21, shape, 7000).cuda()
    before = ops.launch_count()
    out = ops.tt_gather_batch(trains, idx)
    assert ops.launch_count() - before == tm.launches([[1, 3 + b, 20 - b, 2 + b, 1] for b in range(3)], 0, 4, 7000)
    for b in range(3):
        assert_within(out[b], trains[b], idx, 0, 4, torch.float64)


# ------------------------------------------------------------------ reproducibility, cross_tt_eval
def test_bitwise_reproducible_and_shuffle_invariant():
    shape, ranks = [6, 5, 7, 4, 3], [1, 16, 24, 20, 32, 1]
    for dt in DTYPES.values():
        cores = rand_tt(31, shape, ranks, dt)
        idx = rand_idx(32, shape, 20000).cuda()
        a = ops.tt_gather(cores, idx, check=False)
        b = ops.tt_gather(cores, idx, check=False)
        assert torch.equal(a, b)
        perm = torch.randperm(20000, generator=torch.Generator().manual_seed(3)).cuda()
        c = ops.tt_gather(cores, idx[perm], check=False)
        assert torch.equal(c, a[:, perm, :])


def test_agrees_with_cross_tt_eval():
    shape, ranks = [9, 8, 7, 6], [1, 12, 40, 64, 1]
    cores = rand_tt(41, shape, ranks)
    idx = rand_idx(42, shape, 3000).cuda()
    got = ops.tt_gather(cores, idx)[0, :, 0]
    ref = ops.cross_tt_eval([c[None] for c in cores], idx.int())[0]
    absw = tm.gather(np_cores(cores), idx.cpu().numpy(), absolute=True)[0, :, 0]
    K = tm.depth(ranks, 0, 4) + 1
    assert (np.abs((got - ref).cpu().numpy()) <= 8 * K * U[torch.float64] * absw).all()


# ------------------------------------------------------------------ the C-ABI's buffers, streams, synchronisation
def _abi(cores, idx, out, ws, ws_bytes, first=0, last=None):
    last = len(cores) if last is None else last
    shape = [c.shape[1] for c in cores]
    ranks = [cores[0].shape[0]] + [c.shape[2] for c in cores]
    ptrs = (C.c_void_p * len(cores))(*[c.data_ptr() for c in cores])
    code = _lib.TNB_F64 if cores[0].dtype == torch.float64 else _lib.TNB_F32
    return _lib.lib().tnb_tt_gather(code, ptrs, 1, len(cores), _lib.i64(shape), _lib.i32(ranks), first, last,
                                    C.c_void_p(idx.data_ptr()), idx.shape[0], C.c_void_p(out.data_ptr()),
                                    C.c_void_p(ws.data_ptr()), ws_bytes, C.c_void_p(torch.cuda.current_stream().cuda_stream))


@pytest.mark.parametrize("P", [300, 6000])
def test_canaries_and_refusals_leave_out_alone(P):
    shape, ranks = [6, 5, 7, 4], [1, 16, 24, 20, 1]
    cores = rand_tt(51, shape, ranks)
    idx = rand_idx(52, shape, P).cuda()
    L = _lib.lib()
    wsb = L.tnb_tt_gather_workspace_bytes(_lib.TNB_F64, 1, 4, _lib.i64(shape), _lib.i32(ranks), 0, 4, P)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    buf = torch.full((P + 64,), 7.25, dtype=torch.float64, device="cuda")
    out = buf[32:32 + P]
    assert _abi(cores, idx, out, ws, wsb) == 0
    assert (buf[:32] == 7.25).all() and (buf[32 + P:] == 7.25).all()
    assert_within(out[None, :, None], cores, idx, 0, 4, torch.float64)
    buf.fill_(7.25)
    before = ops.launch_count()
    if wsb > 256:
        assert _abi(cores, idx, out, ws, wsb - 1) == _lib.ERR_WORKSPACE
    assert _abi(cores, idx, out, ws, wsb, first=2, last=1) == _lib.ERR_INVALID
    assert ops.launch_count() == before
    torch.cuda.synchronize()
    assert (buf == 7.25).all()


def test_two_streams_on_two_threads():
    shape, ranks = [6, 5, 7, 4, 3], [1, 16, 24, 20, 32, 1]
    cores = rand_tt(61, shape, ranks)
    idxs = [rand_idx(62 + i, shape, 9000).cuda() for i in range(2)]
    want = [ops.tt_gather(cores, ix) for ix in idxs]
    got = [None, None]

    def run(i):
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            for _ in range(5):
                got[i] = ops.tt_gather(cores, idxs[i], check=False)
        s.synchronize()

    th = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for i in range(2):
        assert torch.equal(got[i], want[i])


def test_no_host_synchronisation_with_check_false():
    shape, ranks = [6, 5, 7, 4], [1, 16, 24, 20, 1]
    cores = rand_tt(71, shape, ranks)
    for P in (300, 6000):
        idx = rand_idx(72, shape, P).cuda()
        ops.tt_gather(cores, idx, check=False)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            ops.tt_gather(cores, idx, check=False)
            ops.tt_gather(cores, idx.int(), check=False)
        finally:
            torch.cuda.set_sync_debug_mode(0)


# ------------------------------------------------------------------ keys the kernel must never see
def test_out_of_range_keys_raise_before_any_launch():
    shape, ranks = [6, 5, 7, 4], [1, 3, 4, 2, 1]
    cores = rand_tt(81, shape, ranks)
    t = tn.Tensor(cores)
    for key in (np.array([[0, 0, 0, 4]]), np.array([[0, -6, 0, 0]])):
        for k in (key, torch.tensor(key).cuda()):
            before = ops.launch_count()
            with pytest.raises(IndexError):
                ops.tt_gather(cores, k)
            assert ops.launch_count() == before
    before = ops.launch_count()
    with pytest.raises(IndexError):
        t[torch.tensor([[0, 0, 7, 0]]).cuda()]
    with pytest.raises(IndexError):
        t[1, 2, 3, 4]
    with pytest.raises(IndexError):
        t[[0, 1], [0, 9], 1]
    assert ops.launch_count() == before


def test_getitem_errors_and_gradients():
    shape, ranks = [6, 5, 7, 4], [1, 3, 4, 2, 1]
    t = tn.Tensor(rand_tt(91, shape, ranks))
    with pytest.raises(NotImplementedError):
        t[t]
    tb = tn.Tensor([c[None].repeat(2, 1, 1, 1) for c in rand_tt(92, shape, ranks)], batch=True)
    with pytest.raises(ValueError):
        tb[[0, 1], 1, 2, 3, 0]
    with pytest.raises(ValueError):
        tb[None]
    cores = [c.clone().requires_grad_() for c in rand_tt(93, shape, ranks)]
    tg = tn.Tensor(cores)
    Xs = rand_idx(94, shape, 50)
    v = tg[Xs].torch()
    v.sum().backward()
    ref = tn.Tensor([c.detach() for c in cores])[Xs].torch()
    torch.testing.assert_close(v.detach(), ref, rtol=1e-12, atol=1e-14)
    assert all(c.grad is not None for c in cores)


# ------------------------------------------------------------------ scale
def test_config3_at_2_20_points():
    shape, ranks = [128] * 10, [1] + [64] * 9 + [1]
    cores = rand_tt(101, shape, ranks)
    P = 1 << 20
    idx = rand_idx(102, shape, P).cuda()
    out = ops.tt_gather(cores, idx)[0, :, 0]
    sub = torch.randperm(P, generator=torch.Generator().manual_seed(5))[:4096].cuda()
    assert_within(out[sub][None, :, None], cores, idx[sub], 0, 10, torch.float64)
    from tntorch_b200.cross import _evaluate_tt_at

    for p0 in range(0, P, 1 << 14):
        cols = [idx[p0:p0 + (1 << 14), k] for k in range(10)]
        ref = _evaluate_tt_at(cores, cols)
        torch.testing.assert_close(out[p0:p0 + (1 << 14)], ref, rtol=1e-10, atol=1e-12)


def test_state_past_2_31_elements():
    shape, ranks = [8, 8, 8], [1, 80, 80, 1]
    P = 1 << 25
    need = 2 * P * 80 * 4 + P * 3 * 8 * 2 + P * 4 * 4
    if torch.cuda.mem_get_info()[0] < need + (4 << 30):
        pytest.skip("not enough free device memory for a state past 2^31 elements")
    assert P * 80 > 2 ** 31
    cores = rand_tt(111, shape, ranks, torch.float32)
    idx = rand_idx(112, shape, P).cuda()
    out = ops.tt_gather(cores, idx, check=False)[0, :, 0]
    sub = torch.cat([torch.arange(4096), torch.arange(P - 4096, P)]).cuda()
    assert_within(out[sub][None, :, None], cores, idx[sub], 0, 3, torch.float32)
    del out, idx


def test_rank_256_fp32_on_the_tensor_cores():
    shape, ranks = [16] * 8, [1, 16, 256, 256, 256, 256, 256, 16, 1]
    cores = rand_tt(121, shape, ranks, torch.float32)
    idx = rand_idx(122, shape, 1 << 16).cuda()
    assert tm.mode_paths(ranks, 0, 8).count(tm.TC) == 6
    out = ops.tt_gather(cores, idx)
    sub = torch.arange(0, 1 << 16, 64).cuda()
    assert_within(out[:, sub, :], cores, idx[sub], 0, 8, torch.float32)
