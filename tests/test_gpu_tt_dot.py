"""-m gpu: inner products of tensor trains on the device (tnb_tt_dot through ops.tt_dot / tt_dot_batch, tn.dot, normsq,
norm, dist, the Tensor methods and relative_error(TT, TT)).

- the reference's own results on every case of tests/golden/metrics.npz;
- every branch of the chooser (ttd_mode_path, restated in tests/ttd_model.py) against the fp64 NumPy chain within
  c K 2^-53 <|a|, |b|>, the branch seen in the kernels that run and the launches counted;
- exact results on small-integer cores, bitwise reproducibility, a pair alone against the same pair in a batch of 64;
- canaries around `out`, refusals that leave `out` alone, two streams on two threads, no host synchronisation;
- rank 256, and config 3 (128^10, rank 64): relative_error(t, round_tt(t, rmax=16)) without densifying.
"""
import ctypes as C
import json
import math
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

import ttd_model as tm
from oracle import cases
from test_tt_dot_oracle import GOLD, cfg3_pair, golden_names, golden_pair

pytestmark = pytest.mark.gpu
U53 = 2.0 ** -53

# name -> (shape, inner ranks of a, inner ranks of b): a case for every branch of ttd_mode_path (named by
# ttd_model.BRANCHES); the boundary modes of every case run the generic path
PATH_CASES = {
    "tensor cores": ([6, 5, 7, 4], [16, 24, 20], [20, 16, 32]),
    "a rank below 16": ([3, 4, 5], [3, 4], [2, 5]),
    "a rank above 256": ([4, 3, 5], [4, 300], [4, 270]),
}


def rand_tt(seed, shape, ranks, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    r = [1] + list(ranks) + [1]
    return [torch.randn(r[k], shape[k], r[k + 1], generator=g, dtype=dtype).cuda() for k in range(len(shape))]


def np_cores(cs):
    return [c.detach().cpu().double().numpy() for c in cs]


def ranks_of(cs):
    return [1] + [int(c.shape[2]) for c in cs]


def bound(a, b, c=2.0):
    """c K 2^-53 <|a|, |b|>: the device's rounding and the CPU chain's, each at most K u <|a|, |b|> to first order, K
    the depth of the longest chain of additions (ttd_model.depth)."""
    A, B = np_cores(a), np_cores(b)
    K = tm.depth([x.shape[1] for x in A], ranks_of(a), ranks_of(b))
    return c * K * U53 * tm.abs_dot(A, B)


def kernels(fn):
    """Names of the ttd_ kernels `fn` launches.  Every call ends in ttd_reduce_kernel, so a trace without it came back
    empty: it is taken again, and an empty one is never accepted."""
    from torch.profiler import ProfilerActivity, profile

    fn()  # first-call attribute setup out of the trace
    torch.cuda.synchronize()
    names = set()
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "ttd_" in e.name}
        if any("ttd_reduce_kernel" in n for n in names):
            break
    assert any("ttd_reduce_kernel" in n for n in names), "the profiler recorded no ttd_ kernel"
    return sorted(names)


DTYPES = {"float64": torch.float64, "float32": torch.float32}


def trace_path_cases():
    """{"name/dtype": kernel names} of one ops.tt_dot per PATH_CASES entry and dtype; run in a process of its own."""
    from tntorch_b200 import ops

    out = {}
    for name, (shape, ra, rb) in PATH_CASES.items():
        for dn, dt in DTYPES.items():
            a, b = rand_tt(1, shape, ra, dt), rand_tt(2, shape, rb, dt)
            out[f"{name}/{dn}"] = kernels(lambda: ops.tt_dot(a, b))
    return out


@pytest.fixture(scope="module")
def path_kernels():
    """The kernels of every path case, traced in a fresh process: late in a long process that has profiled before, the
    activity trace has come back without some of the kernels a call launched."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here, os.environ.get("PYTHONPATH", "")]))
    code = "import json, test_gpu_tt_dot as t; print('TRACE ' + json.dumps(t.trace_path_cases()))"
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=os.path.dirname(here),
                       timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    line = [x for x in r.stdout.splitlines() if x.startswith("TRACE ")][-1]
    return json.loads(line[len("TRACE "):])


# ------------------------------------------------------------------ the reference's results
@pytest.mark.parametrize("name", golden_names())
def test_matches_reference(name):
    import tntorch_b200 as tnb

    g = np.load(GOLD)
    ((ca, Ua), (cb, Ub)), dt = golden_pair(g, name)

    def tensor(cs, Us):
        return tnb.Tensor([torch.from_numpy(c).cuda() for c in cs],
                          Us=None if all(u is None for u in Us) else [None if u is None else torch.from_numpy(u).cuda() for u in Us])

    a, b = tensor(ca, Ua), tensor(cb, Ub)
    got = dict(dot=tnb.dot(a, b), normsq_a=tnb.normsq(a), norm_a=tnb.norm(a), norm_b=b.norm(), dist=tnb.dist(a, b),
               relerr=tnb.relative_error(a, b))
    assert got["dot"].dtype == torch.float64 and got["dot"].dim() == 0 and got["dot"].is_cuda
    assert float(a.dot(b)) == float(got["dot"]) and float(a.normsq()) == float(got["normsq_a"])
    rtol = 2e-5 if dt == np.float32 else 1e-12
    na, nb = float(g[f"{name}/norm_a"]), float(g[f"{name}/norm_b"])
    for key, v in got.items():
        ref = float(g[f"{name}/{key}"])
        scale = {"dot": na * nb, "normsq_a": na * na}.get(key, abs(ref))
        assert abs(float(v) - ref) <= rtol * scale, (name, key, float(v), ref)


# ------------------------------------------------------------------ every path against the fp64 chain
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("name", list(PATH_CASES))
def test_path_against_fp64_chain(name, dtype, path_kernels):
    from tntorch_b200 import ops

    shape, ra, rb = PATH_CASES[name]
    a, b = rand_tt(1, shape, ra, dtype), rand_tt(2, shape, rb, dtype)
    want = tm.dot(np_cores(a), np_cores(b))
    n0 = ops.launch_count()
    got = ops.tt_dot(a, b)
    assert ops.launch_count() - n0 == tm.launches(shape, [ranks_of(a)], [ranks_of(b)])
    assert abs(float(got) - want) <= bound(a, b), (float(got), want)
    used = set(tm.paths(shape, [ranks_of(a)], [ranks_of(b)])[0])
    names = path_kernels[f"{name}/{str(dtype).replace('torch.', '')}"]
    assert any("ttd_mode_tc_kernel" in k for k in names) == (tm.TC in used), names
    assert any("ttd_mode_generic_kernel" in k for k in names) == bool(used - {tm.TC}), names
    # the norm: the same cores for a and b
    aa = ops.tt_dot(a, a)
    assert abs(float(aa) - tm.dot(np_cores(a), np_cores(a))) <= bound(a, a)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_small_integers_are_exact(dtype):
    """Cores in {-1, 0, 1}: every partial sum is an integer below 2^53, so the result is exact on both paths."""
    from tntorch_b200 import ops

    shape, ra, rb = [4, 5, 6, 3], [16, 20, 24], [20, 16, 17]
    g = torch.Generator().manual_seed(7)

    def ints(r):
        r = [1] + r + [1]
        return [torch.randint(-1, 2, (r[k], shape[k], r[k + 1]), generator=g).to(dtype).cuda() for k in range(len(shape))]

    a, b = ints(ra), ints(rb)
    assert tm.TC in tm.paths(shape, [ranks_of(a)], [ranks_of(b)])[0]
    f = np.ones((1, 1), dtype=np.int64)
    for x, y in zip(a, b):
        f = np.einsum("ab,aic,bid->cd", f, x.cpu().numpy().astype(np.int64), y.cpu().numpy().astype(np.int64))
    assert float(ops.tt_dot(a, b)) == float(f[0, 0])


# ------------------------------------------------------------------ determinism, batches
def test_bitwise_reproducible_and_batch_agrees():
    from tntorch_b200 import ops

    shape = [32] * 6
    pairs = [(rand_tt(100 + p, shape, [32] * 5), rand_tt(200 + p, shape, [16, 32, 48, 32, 16])) for p in range(64)]
    x = ops.tt_dot_batch(pairs)
    y = ops.tt_dot_batch(pairs)
    assert x.shape == (64,) and torch.equal(x, y)
    for p in (0, 17, 63):
        a, b = pairs[p]
        alone = ops.tt_dot(a, b)
        assert abs(float(alone) - float(x[p])) <= bound(a, b), p
        assert torch.equal(alone, ops.tt_dot(a, b))


def test_batched_tensors_take_one_call():
    import tntorch_b200 as tnb
    from tntorch_b200 import ops

    shape, B = [5, 6, 7], 3
    a = [rand_tt(300 + s, shape, [4, 20]) for s in range(B)]
    b = [rand_tt(400 + s, shape, [18, 3]) for s in range(B)]
    ta = tnb.Tensor([torch.stack([x[k] for x in a]) for k in range(3)], batch=True)
    tb = tnb.Tensor([torch.stack([x[k] for x in b]) for k in range(3)], batch=True)
    n0 = ops.launch_count()
    d = tnb.dot(ta, tb)
    assert ops.launch_count() - n0 == tm.launches(shape, [ranks_of(x) for x in a], [ranks_of(x) for x in b])
    assert d.shape == (B,)
    for s in range(B):
        assert abs(float(d[s]) - tm.dot(np_cores(a[s]), np_cores(b[s]))) <= bound(a[s], b[s])
    assert torch.allclose(tnb.norm(ta), torch.stack([ops.tt_dot(x, x) for x in a]).clamp(min=0).sqrt(), rtol=1e-13)
    assert tnb.normsq(ta).shape == (B,) and tnb.dist(ta, tb).shape == (B,)


def test_errors():
    import tntorch_b200 as tnb

    a = tnb.Tensor(rand_tt(1, [3, 4, 5], [2, 2]))
    with pytest.raises(NotImplementedError):
        tnb.dot(a, a, k=1)
    with pytest.raises(NotImplementedError):
        tnb.dot(a, tnb.Tensor(rand_tt(1, [3, 4], [2])))
    with pytest.raises(ValueError):
        tnb.dot(a, tnb.Tensor(rand_tt(1, [3, 4, 6], [2, 2])))
    with pytest.raises(ValueError):
        tnb.dist(a, tnb.Tensor(rand_tt(1, [3, 5, 5], [2, 2])))


# ------------------------------------------------------------------ isolation
def _raw_call(a, b, out, ws_bytes=None, ranks_a=None):
    from tntorch_b200 import _lib, ops

    L = _lib.lib()
    shape = [c.shape[1] for c in a]
    sh, ra, rb = _lib.i64(shape), _lib.i32(ranks_a or ranks_of(a)), _lib.i32(ranks_of(b))
    wsb = L.tnb_tt_dot_workspace_bytes(_lib.TNB_F64, 1, len(a), sh, ra, rb)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    pa = (C.c_void_p * len(a))(*[c.data_ptr() for c in a])
    pb = (C.c_void_p * len(b))(*[c.data_ptr() for c in b])
    return L.tnb_tt_dot(_lib.TNB_F64, pa, pb, 1, len(a), sh, ra, rb, C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()),
                        wsb if ws_bytes is None else ws_bytes, ops._stream())


def test_canaries_and_refusals_leave_out_alone():
    from tntorch_b200 import _lib

    a, b = rand_tt(5, [6, 5, 7, 4], [16, 24, 20]), rand_tt(6, [6, 5, 7, 4], [20, 16, 32])
    buf = torch.full((3,), 12345.0, dtype=torch.float64, device="cuda")
    assert _raw_call(a, b, buf[1:2]) == 0
    torch.cuda.synchronize()
    assert float(buf[0]) == 12345.0 and float(buf[2]) == 12345.0 and float(buf[1]) != 12345.0
    buf.fill_(12345.0)
    assert _raw_call(a, b, buf[1:2], ws_bytes=64) == _lib.ERR_WORKSPACE
    assert _raw_call(a, b, buf[1:2], ranks_a=[2] + ranks_of(a)[1:]) == _lib.ERR_INVALID  # boundary rank 2
    torch.cuda.synchronize()
    assert torch.equal(buf, torch.full_like(buf, 12345.0))


def test_two_streams_on_two_threads_and_no_host_sync():
    from tntorch_b200 import ops

    work = [(rand_tt(10 + t, [16] * 5, [24] * 4), rand_tt(20 + t, [16] * 5, [20] * 4)) for t in range(2)]
    want = [ops.tt_dot(a, b) for a, b in work]
    got = [None, None]

    def run(t):
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            r = [ops.tt_dot(*work[t]) for _ in range(5)]
        s.synchronize()
        got[t] = r

    th = [threading.Thread(target=run, args=(t,)) for t in range(2)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    for t in range(2):
        assert all(torch.equal(r, want[t]) for r in got[t])
    torch.cuda.set_sync_debug_mode("error")
    try:
        ops.tt_dot_batch(work)
    finally:
        torch.cuda.set_sync_debug_mode(0)


# ------------------------------------------------------------------ rank 256 and config 3
def test_rank_256():
    from tntorch_b200 import ops

    shape = [16] * 5
    a, b = rand_tt(31, shape, [16, 256, 256, 16]), rand_tt(32, shape, [16, 256, 200, 16])
    assert tm.TC in tm.paths(shape, [ranks_of(a)], [ranks_of(b)])[0]
    got = ops.tt_dot(a, b)
    assert abs(float(got) - tm.dot(np_cores(a), np_cores(b))) <= bound(a, b)


def _einsum_dot(a, b):
    m = torch.ones(1, 1, dtype=torch.float64, device=a[0].device)
    for x, y in zip(a, b):
        m = torch.einsum("ab,aic,bid->cd", m, x.double(), y.double())
    return float(m[0, 0])


def test_config3_relative_error_without_densifying():
    import tntorch_b200 as tnb
    from tntorch_b200 import ops

    spec = cases.FULL_ROUND_CASES["cfg3_128x10_r64to16_f64"]
    t = tnb.Tensor([torch.as_tensor(c).cuda() for c in cases.make_tt(spec)])
    r = tnb.round_tt(t, rmax=spec["rmax"])
    err = tnb.relative_error(t, r)
    ref = float(np.load(os.path.join(os.path.dirname(GOLD), "full.npz"))["cfg3_128x10_r64to16_f64/svd/relerr"])
    assert abs(err - ref) <= 1e-7, (err, ref)
    aa, rr, ar = ops.tt_dot_batch([(t.cores, t.cores), (r.cores, r.cores), (t.cores, r.cores)])
    ea, er, ex = _einsum_dot(t.cores, t.cores), _einsum_dot(r.cores, r.cores), _einsum_dot(t.cores, r.cores)
    assert abs(float(aa) - ea) <= 1e-12 * ea and abs(float(rr) - er) <= 1e-12 * er
    assert abs(float(ar) - ex) <= 1e-12 * math.sqrt(ea * er)


def test_config3_matches_reference():
    import tntorch_b200 as tnb

    g = np.load(GOLD)
    ca, cb = cfg3_pair(g)
    a, b = tnb.Tensor([torch.as_tensor(c).cuda() for c in ca]), tnb.Tensor([torch.as_tensor(c).cuda() for c in cb])
    na, nb = float(g["cfg3/norm_a"]), float(g["cfg3/norm_b"])
    got = dict(dot=tnb.dot(a, b), normsq_a=tnb.normsq(a), norm_a=tnb.norm(a), norm_b=tnb.norm(b), dist=tnb.dist(a, b),
               relerr=tnb.relative_error(a, b))
    for key, v in got.items():
        ref = float(g[f"cfg3/{key}"])
        scale = {"dot": na * nb, "normsq_a": na * na}.get(key, abs(ref))
        assert abs(float(v) - ref) <= 1e-12 * scale, (key, float(v), ref)
