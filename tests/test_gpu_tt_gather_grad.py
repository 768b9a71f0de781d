"""-m gpu: the gradient of entries of tensor trains (tnb_tt_gather_grad through ops.tt_gather / tt_gather_batch under
autograd and Tensor.__getitem__).

- the reference's own gradients on every value case of tests/golden/getitem_grad.npz (TT, Tucker, TT-Tucker, CP, batch);
- every branch of the backward (tests/ttgg_model.py) in both dtypes against the fp64 torch chain's autograd within
  c K u (the gradient in absolute values), the kernels read from a profiler trace and the launches counted;
- torch.autograd.gradcheck through ops.tt_gather and t[Xs]; bitwise reproducibility; no host synchronisation;
  points with an out-of-range index excluded; canaries, refusals and two streams at the C-ABI;
- config 3 at P = 2^20 against chunked fp64 chain gradients; an Adam fit against the same fit through the chain.
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
import ttgg_model as gm
from oracle import getitem_cases as gc
from tntorch_b200 import _lib, ops
from test_getitem_oracle import GOLD

pytestmark = pytest.mark.gpu
GOLD_GRAD = os.path.join(os.path.dirname(__file__), "golden", "getitem_grad.npz")
U = {torch.float64: 2.0 ** -53, torch.float32: 2.0 ** -24}
DTYPES = {"float64": torch.float64, "float32": torch.float32}

# name -> (shape, ranks, first, last, P): every branch of the backward
BRANCH_CASES = {
    "tensor cores": ([6, 5, 7, 4, 3], [1, 16, 24, 20, 32, 1], 0, 5, 6000),
    "generic": ([5, 9, 3], [1, 4, 7, 1], 0, 3, 9000),
    "a rank above 256": ([4, 3, 5], [1, 20, 300, 1], 0, 3, 3000),
    "one mode": ([11], [1, 1], 0, 1, 5000),
    "inner range, r_first and r_last above 1": ([6, 5, 7, 4, 3], [1, 16, 24, 20, 32, 1], 1, 4, 3000),
    "first mode on the tensor cores": ([6, 5, 7], [16, 16, 24, 16], 0, 3, 2000),
    "unused index values": ([300, 5, 7], [1, 16, 16, 1], 0, 3, 100),
    "multi-chunk buckets": ([2] * 8, [1] + [16] * 7 + [1], 0, 8, 20000),
    "multi-chunk buckets, generic": ([2] * 6, [1, 3, 5, 4, 2, 3, 1], 0, 6, 30000),
}


def rand_tt(seed, shape, ranks, dtype=torch.float64, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(ranks[k], shape[k], ranks[k + 1], generator=g, dtype=torch.float64) / ranks[k] ** 0.5)
            .to(dtype).to(device) for k in range(len(shape))]


def rand_idx(seed, shape, P, first=0, last=None):
    last = len(shape) if last is None else last
    g = torch.Generator().manual_seed(seed)
    return torch.stack([torch.randint(0, shape[k], (P,), generator=g) for k in range(first, last)], dim=1)


def chain(cores, idx, first, last):
    """The reference's chain of core[:, idx, :] products (torch, differentiable)."""
    s = cores[first][:, idx[:, 0], :]
    for m, k in enumerate(range(first + 1, last), start=1):
        s = torch.einsum("iaj,jak->iak", s, cores[k][:, idx[:, m], :])
    return s


def library_grads(cores, idx, first, last, w, check=False):
    leaves = [c.detach().clone().requires_grad_() for c in cores]
    out = ops.tt_gather(leaves, idx, first, last, check=check)
    (out * w).sum().backward()
    return [leaves[k].grad for k in range(first, last)]


def assert_grads_within(got, cores, idx, first, last, w, dtype, c=4.0):
    """|got - chain autograd| <= c K u |grad|_abs, K = the chain's depth and both boundary ranks plus the rows of a
    chunk and the chunks of a bucket."""
    leaves = [c_.detach().double().clone().requires_grad_() for c_ in cores]
    (chain(leaves, idx, first, last) * w.double()).sum().backward()
    A = [c_.detach().cpu().double().numpy() for c_ in cores]
    absg = gm.grad(A, idx.cpu().numpy(), w.detach().cpu().double().numpy(), first, last, absolute=True)
    ranks = [A[0].shape[0]] + [a.shape[2] for a in A]
    P = idx.shape[0]
    for m, k in enumerate(range(first, last)):
        rows = P * ranks[first]
        ch = gm.chunk_rows(rows, ranks[k], ranks[k + 1])
        K = tm.depth(ranks, first, last) + ranks[first] + ranks[last] + ch + -(-rows // ch)
        err = np.abs(got[m].detach().cpu().double().numpy() - leaves[k].grad.cpu().numpy())
        lim = c * K * U[dtype] * absg[m] + 1e-300
        assert (err <= lim).all(), (k, float((err / lim).max()))


def kernels(fn):
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                   and ("ttgg_" in e.name or "ttg_step" in e.name)})


def trace_branch_cases():
    """{"name/dtype": kernel names} of one backward per BRANCH_CASES entry and dtype; run in a process of its own."""
    out = {}
    for name, (shape, ranks, first, last, P) in BRANCH_CASES.items():
        for dn, dt in DTYPES.items():
            cores = rand_tt(11, shape, ranks, dt)
            idx = rand_idx(12, shape, P, first, last).cuda()
            leaves = [c.requires_grad_() for c in cores]
            out[f"{name}/{dn}"] = kernels(lambda: ops.tt_gather(leaves, idx, first, last, check=False).sum().backward())
    return out


@pytest.fixture(scope="module")
def branch_kernels():
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here, os.environ.get("PYTHONPATH", "")]))
    code = "import json, test_gpu_tt_gather_grad as t; print('TRACE ' + json.dumps(t.trace_branch_cases()))"
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=os.path.dirname(here),
                       timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    line = [x for x in r.stdout.splitlines() if x.startswith("TRACE ")][-1]
    return json.loads(line[len("TRACE "):])


# ------------------------------------------------------------------ every branch against the fp64 chain's autograd
@pytest.mark.parametrize("dname", list(DTYPES))
@pytest.mark.parametrize("case", list(BRANCH_CASES))
def test_branch(case, dname, branch_kernels):
    dt = DTYPES[dname]
    shape, ranks, first, last, P = BRANCH_CASES[case]
    cores = rand_tt(11, shape, ranks, dt)
    idx = rand_idx(12, shape, P, first, last).cuda()
    w = torch.randn(ranks[first], P, ranks[last], generator=torch.Generator().manual_seed(13), dtype=torch.float64)
    w = w.to(dt).cuda()
    leaves = [c.detach().clone().requires_grad_() for c in cores]
    out = ops.tt_gather(leaves, idx, first, last, check=False)
    loss = (out * w).sum()
    before = ops.launch_count()
    loss.backward()
    torch.cuda.synchronize()
    bwd = ops.launch_count() - before
    # the backward's own launches, plus the loss's (mul, sum and their backward run on torch kernels, not counted)
    assert bwd == gm.launches(shape, [ranks], first, last), (bwd, gm.launches(shape, [ranks], first, last))
    got = [leaves[k].grad for k in range(first, last)]
    assert all(g.dtype == dt and g.shape == cores[k].shape for g, k in zip(got, range(first, last)))
    assert all(leaves[k].grad is None for k in range(len(shape)) if not first <= k < last)
    assert_grads_within(got, cores, idx, first, last, w, dt)
    names = branch_kernels[f"{case}/{dname}"]
    seen = {k for k in ("ttgg_reduce_tc_kernel", "ttgg_reduce_generic_kernel", "ttg_step_tc_kernel",
                        "ttg_step_generic_kernel") if any(k in n and ("true" in n or "ttgg" in k) for n in names)}
    assert seen == gm.kernels(ranks, first, last), (names, gm.kernels(ranks, first, last))
    if case == "unused index values":
        used = set(idx[:, 0].tolist())
        unused = [i for i in range(shape[0]) if i not in used]
        assert unused and (got[0][:, unused, :] == 0).all()
    if case.startswith("multi-chunk"):
        rows = P * ranks[first]
        assert rows // 2 > gm.chunk_rows(rows, ranks[1], ranks[2])


def test_duplicate_points_and_several_trains():
    shape = [6, 5, 7, 4]
    rks = [[1, 3 + b, 20 - b, 2 + b, 1] for b in range(3)]
    trains = [rand_tt(20 + b, shape, rks[b]) for b in range(3)]
    idx = rand_idx(21, shape, 3000)
    idx = torch.cat([idx, idx[:1000], idx[:500]]).cuda()  # duplicates
    P = idx.shape[0]
    w = torch.randn(3, 1, P, 1, generator=torch.Generator().manual_seed(22), dtype=torch.float64).cuda()
    leaves = [[c.clone().requires_grad_() for c in t] for t in trains]
    out = ops.tt_gather_batch(leaves, idx, check=False)
    before = ops.launch_count()
    (out * w).sum().backward()
    torch.cuda.synchronize()
    assert ops.launch_count() - before == gm.launches(shape, rks, 0, 4)
    for b in range(3):
        assert_grads_within([c.grad for c in leaves[b]], trains[b], idx, 0, 4, w[b], torch.float64)


# ------------------------------------------------------------------ gradcheck, reproducibility, synchronisation
def test_gradcheck_through_tt_gather_and_getitem():
    shape, ranks = [4, 3, 5], [2, 3, 2, 2]
    cores = [c.requires_grad_() for c in rand_tt(31, shape, ranks)]
    idx = rand_idx(32, shape, 40).cuda()
    assert torch.autograd.gradcheck(lambda *cs: ops.tt_gather(list(cs), idx, check=False), cores)
    cores = [c.detach().requires_grad_() for c in rand_tt(33, shape, [1, 3, 2, 1])]
    Xs = rand_idx(34, shape, 30)
    assert torch.autograd.gradcheck(lambda *cs: tn.Tensor(list(cs))[Xs].torch(), cores)
    g = ops.tt_gather(cores, idx[:, :3], check=False)
    (gr,) = torch.autograd.grad(g.sum(), cores[0], create_graph=True)
    with pytest.raises(RuntimeError):
        gr.sum().backward()


def test_bitwise_reproducible():
    shape, ranks = [6, 5, 7, 4, 3], [1, 16, 24, 20, 32, 1]
    for dt in DTYPES.values():
        cores = rand_tt(41, shape, ranks, dt)
        idx = rand_idx(42, shape, 20000).cuda()
        w = torch.randn(1, 20000, 1, generator=torch.Generator().manual_seed(43)).to(dt).cuda()
        a = library_grads(cores, idx, 0, 5, w)
        b = library_grads(cores, idx, 0, 5, w)
        assert all(torch.equal(x, y) for x, y in zip(a, b))
    shape, ranks = [2] * 8, [1] + [16] * 7 + [1]
    cores = rand_tt(44, shape, ranks, torch.float32)
    idx = rand_idx(45, shape, 1 << 16).cuda()
    w = torch.randn(1, 1 << 16, 1, generator=torch.Generator().manual_seed(46)).cuda()
    a = library_grads(cores, idx, 0, 8, w)
    b = library_grads(cores, idx, 0, 8, w)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_no_host_synchronisation_in_backward():
    shape, ranks = [6, 5, 7, 4], [1, 16, 24, 20, 1]
    cores = [c.requires_grad_() for c in rand_tt(51, shape, ranks)]
    idx = rand_idx(52, shape, 6000).cuda()
    ops.tt_gather(cores, idx, check=False).sum().backward()
    torch.cuda.synchronize()
    out = ops.tt_gather(cores, idx, check=False)
    gout = torch.ones_like(out)
    torch.cuda.set_sync_debug_mode("error")
    try:
        torch.autograd.backward(out, gout)
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_out_of_range_points_are_excluded():
    shape, ranks = [6, 5, 7, 4], [1, 16, 24, 20, 1]
    cores = rand_tt(61, shape, ranks)
    idx = rand_idx(62, shape, 5000)
    bad = torch.cat([idx[:2000], torch.tensor([[1, 7, 2, 0]]), idx[2000:]]).cuda()
    w = torch.randn(1, 5001, 1, generator=torch.Generator().manual_seed(63), dtype=torch.float64).cuda()
    got = library_grads(cores, bad, 0, 4, w)
    want = library_grads(cores, idx.cuda(), 0, 4, torch.cat([w[:, :2000], w[:, 2001:]], dim=1))
    for g, h in zip(got, want):
        torch.testing.assert_close(g, h, rtol=1e-13, atol=1e-15)


# ------------------------------------------------------------------ the C-ABI's buffers and streams
def _abi(cores, idx, gout, grads, ws, ws_bytes, first=0, last=None):
    last = len(cores) if last is None else last
    shape = [c.shape[1] for c in cores]
    ranks = [cores[0].shape[0]] + [c.shape[2] for c in cores]
    ptrs = (C.c_void_p * len(cores))(*[c.data_ptr() for c in cores])
    gptrs = (C.c_void_p * len(cores))(*[g.data_ptr() for g in grads])
    code = _lib.TNB_F64 if cores[0].dtype == torch.float64 else _lib.TNB_F32
    return _lib.lib().tnb_tt_gather_grad(code, ptrs, 1, len(cores), _lib.i64(shape), _lib.i32(ranks), first, last,
                                         C.c_void_p(idx.data_ptr()), idx.shape[0], C.c_void_p(gout.data_ptr()), gptrs,
                                         C.c_void_p(ws.data_ptr()), ws_bytes,
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream))


def test_canaries_and_refusals_leave_grads_alone():
    shape, ranks, P = [6, 5, 7, 4], [1, 16, 24, 20, 1], 6000
    cores = rand_tt(71, shape, ranks)
    idx = rand_idx(72, shape, P).cuda()
    gout = torch.randn(1, P, 1, generator=torch.Generator().manual_seed(73), dtype=torch.float64).cuda()
    L = _lib.lib()
    wsb = L.tnb_tt_gather_grad_workspace_bytes(_lib.TNB_F64, 1, 4, _lib.i64(shape), _lib.i32(ranks), 0, 4, P)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    bufs = [torch.full((c.numel() + 64,), 7.25, dtype=torch.float64, device="cuda") for c in cores]
    grads = [b[32:32 + c.numel()].view(c.shape) for b, c in zip(bufs, cores)]
    assert _abi(cores, idx, gout, grads, ws, wsb) == 0
    want = library_grads(cores, idx, 0, 4, gout)
    for b, g, h in zip(bufs, grads, want):
        assert (b[:32] == 7.25).all() and (b[-32:] == 7.25).all()
        assert torch.equal(g, h)
    for b in bufs:
        b.fill_(7.25)
    before = ops.launch_count()
    assert _abi(cores, idx, gout, grads, ws, wsb - 1) == _lib.ERR_WORKSPACE
    assert _abi(cores, idx, gout, grads, ws, wsb, first=2, last=1) == _lib.ERR_INVALID
    assert ops.launch_count() == before
    torch.cuda.synchronize()
    assert all((b == 7.25).all() for b in bufs)


def test_two_streams_on_two_threads():
    shape, ranks = [6, 5, 7, 4, 3], [1, 16, 24, 20, 32, 1]
    cores = rand_tt(81, shape, ranks)
    idxs = [rand_idx(82 + i, shape, 9000).cuda() for i in range(2)]
    w = torch.ones(1, 9000, 1, dtype=torch.float64, device="cuda")
    want = [library_grads(cores, ix, 0, 5, w) for ix in idxs]
    got = [None, None]

    def run(i):
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            for _ in range(3):
                got[i] = library_grads(cores, idxs[i], 0, 5, w)
        s.synchronize()

    th = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for i in range(2):
        assert all(torch.equal(a, b) for a, b in zip(got[i], want[i]))


# ------------------------------------------------------------------ the reference's gradients through __getitem__
def _tensor(g, spec, dname):
    t = gc.tensor(spec, gc.DTYPES[dname])
    if t is None:
        n = int(g[f"{spec}/{dname}/n"])
        cores = [torch.tensor(g[f"{spec}/{dname}/core{k}"]).cuda().requires_grad_() for k in range(n)]
        Us = [torch.tensor(g[f"{spec}/{dname}/U{k}"]).cuda().requires_grad_() for k in range(n)]
        return cores, Us, False
    cores, _, batch = t
    return [c.cuda().requires_grad_() for c in cores], None, batch


def dense(r):
    """r.torch() with Tucker factors absorbed by torch einsums, so that autograd reaches both cores and factors."""
    if all(U is None for U in r.Us):
        return r.torch()
    cores = [c if U is None else torch.einsum("...ijk,...aj->...iak", c, U) for c, U in zip(r.cores, r.Us)]
    return tn.Tensor(cores, batch=r.batch).torch()


GRAD_CASES = [(n, d) for d in gc.DTYPES for n in gc.KEYS if f"{n}/{d}/w" in np.load(GOLD_GRAD).files]


@pytest.mark.parametrize("name,dname", GRAD_CASES)
def test_golden_gradients(name, dname):
    g, gg = np.load(GOLD), np.load(GOLD_GRAD)
    spec, key = gc.KEYS[name]
    cores, Us, batch = _tensor(g, spec, dname)
    t = tn.Tensor(cores, Us=Us, batch=batch)
    r = t[key("cuda")]
    v = dense(r) if isinstance(r, tn.Tensor) else r
    w = torch.as_tensor(gg[f"{name}/{dname}/w"]).cuda()
    (w * v).sum().backward()
    tol = 1e-11 if dname == "f64" else 2e-5
    pairs = [(c, f"dcore{k}") for k, c in enumerate(cores)] + [(u, f"dU{k}") for k, u in enumerate(Us or [])]
    for x, nm in pairs:
        want = gg[f"{name}/{dname}/{nm}"]
        got = (x.grad if x.grad is not None else torch.zeros_like(x)).detach().cpu().double().numpy()
        assert got.shape == want.shape, (nm, got.shape, want.shape)
        assert np.abs(got - want).max() <= tol * max(1.0, np.abs(want).max()), nm


# ------------------------------------------------------------------ scale, end to end
def test_config3_at_2_20_points():
    shape, ranks = [128] * 10, [1] + [64] * 9 + [1]
    cores = rand_tt(91, shape, ranks)
    P = 1 << 20
    idx = rand_idx(92, shape, P).cuda()
    w = torch.randn(1, P, 1, generator=torch.Generator().manual_seed(93), dtype=torch.float64).cuda()
    got = library_grads(cores, idx, 0, 10, w)
    leaves = [c.detach().clone().requires_grad_() for c in cores]
    step = 1 << 15
    for p0 in range(0, P, step):
        (chain(leaves, idx[p0:p0 + step], 0, 10) * w[:, p0:p0 + step]).sum().backward()
    for g, c in zip(got, leaves):
        scale = c.grad.abs().max().item()
        assert (g - c.grad).abs().max().item() <= 1e-9 * scale


def test_adam_fit_matches_the_chain():
    """A rank-4 TT fitted by Adam to 10% of the entries of a 32^4 rank-4 tensor: the loss trajectory over 20 steps
    through the library matches the same fit through the torch chain within 1e-9 relative."""
    shape, ranks = [32] * 4, [1, 4, 4, 4, 1]
    truth = rand_tt(101, shape, ranks)
    P = 32 ** 4 // 10
    idx = rand_idx(102, shape, P).cuda()
    y = ops.tt_gather(truth, idx)[0, :, 0]

    def fit(evaluate):
        cores = [c.clone().requires_grad_() for c in rand_tt(103, shape, ranks)]
        opt = torch.optim.Adam(cores, lr=0.02)
        losses = []
        for _ in range(20):
            opt.zero_grad()
            loss = ((evaluate(cores) - y) ** 2).mean()
            loss.backward()
            opt.step()
            losses.append(loss.item())
        return np.array(losses)

    ours = fit(lambda cs: tn.Tensor(cs)[idx].torch())
    ref = fit(lambda cs: chain(cs, idx, 0, 4)[0, :, 0])
    assert ours[-1] < ours[0]
    np.testing.assert_allclose(ours, ref, rtol=1e-9)
