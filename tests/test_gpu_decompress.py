"""TT -> dense in one library call (tnb_tt_decompress, ops.tt_decompress, Tensor.torch(dtype=, out=)), path by path
against the fp64 chain on the same cores: the split chooser, the tensor-core product inside its envelope and the generic
product outside it, fp32 / bf16 / fp16 / fp64 output, caller-owned buffers, streams, and the C-ABI's bounds.

The dispatch is restated here (split_bond, fast_envelope) and checked against the case list without a GPU; on the GPU
every case asserts the number of launches its restated path implies, so a case cannot silently take another path."""
import ctypes
import math
import threading

import pytest
import torch

from oracle import cases

gpu = pytest.mark.gpu
MIN_ELEMS = 1 << 20   # EXPAND_TC_MIN_ELEMS


# ---------------------------------------------------------------------------------------------- the dispatch, restated
def split_bond(shape, ranks):
    """decompress_split: the bond k in [1, N-1] with the smallest r_k (I_0 .. I_{k-1} + I_k .. I_{N-1}), the last of equals."""
    best, best_k = None, 1
    for k in range(1, len(shape)):
        cost = ranks[k] * (math.prod(shape[:k]) + math.prod(shape[k:]))
        if best is None or cost <= best:
            best, best_k = cost, k
    return best_k


def product_dims(shape, ranks):
    k = split_bond(shape, ranks)
    return k, math.prod(shape[:k]), ranks[k], math.prod(shape[k:])


def fast_envelope(shape, ranks, dtype):
    """expand_tc_shape_ok on the final product of the chosen split (and fp32 cores)."""
    if len(shape) < 2 or dtype != "float32":
        return False
    _, M, K, Nc = product_dims(shape, ranks)
    return 8 <= K <= 256 and Nc % 8 == 0 and M * Nc >= MIN_ELEMS


def expected_launches(shape, ranks, dtype):
    """One launch per chain step, then the product: two split kernels and the tile kernel, or one generic product."""
    N = len(shape)
    if N == 1:
        return 1
    return (N - 2) + (3 if fast_envelope(shape, ranks, dtype) else 1)


# name: (shape, inner ranks, dtype, path, what the case is there for)
CASES = {
    "fast_k8_first_bond": ((128, 128, 64), [8, 8], "float32", "fast", "K=8; k at the first bond"),
    "fast_k32_5d": ((16,) * 5, [32] * 4, "float32", "fast", "K=32; N=5; a tie of two bonds"),
    "fast_k50_padded": ((40, 50, 60, 24), [40, 50, 24], "float32", "fast", "K=50 padded; M, Nc not multiples of the tile"),
    "fast_k64_last_bond": ((128, 96, 128), [64, 64], "float32", "fast", "K=64; N=3; k at the last bond"),
    "fast_k200": ((200, 40, 200), [200, 200], "float32", "fast", "K=200"),
    "fast_k256": ((256, 16, 256), [256, 256], "float32", "fast", "K=256"),
    "fast_n2": ((1024, 1024), [32], "float32", "fast", "N=2"),
    "fast_n8": ((6,) * 8, [12] * 7, "float32", "fast", "N=8; K=12"),
    "generic_k257": ((260, 16, 264), [257, 257], "float32", "generic", "r_k=257"),
    "generic_k4": ((128, 128, 64), [4, 4], "float32", "generic", "r_k below 8"),
    "generic_ragged_nc": ((128, 127, 65), [16, 16], "float32", "generic", "Nc not a multiple of 8"),
    "generic_tiny": ((4, 5, 6), [3, 3], "float32", "generic", "below the element floor"),
    "generic_f64": ((16,) * 5, [32] * 4, "float64", "generic", "fp64 cores"),
    "generic_f64_ragged": ((7, 12, 5, 9, 6), [3, 8, 6, 2], "float64", "generic", "fp64 cores, ragged"),
    "single_n1": ((1000,), [], "float32", "single", "N=1"),
    "single_n1_f64": ((37,), [], "float64", "single", "N=1, fp64"),
}


def test_dispatch_coverage():
    """CPU: the restated chooser and envelope put every case on the path it is listed for, every branch has a case, and
    64^5 at rank 32 splits in the middle."""
    for name, (shape, inner, dtype, path, _) in CASES.items():
        ranks = [1] + inner + [1]
        got = "single" if len(shape) == 1 else "fast" if fast_envelope(shape, ranks, dtype) else "generic"
        assert got == path, name
    dims = {n: product_dims(c[0], [1] + c[1] + [1]) for n, c in CASES.items() if len(c[0]) > 1}
    fast = {n: d for n, d in dims.items() if CASES[n][3] == "fast"}
    assert {8, 32, 50, 64, 200, 256} <= {d[2] for d in fast.values()}
    assert any(d[2] % 8 for d in fast.values())                                      # K padded to a k-step
    assert any(d[1] % 128 and d[3] % 128 for d in fast.values())                     # edge tiles both ways
    assert any(d[0] == 1 for d in fast.values()) and any(d[0] == len(CASES[n][0]) - 1 and d[0] > 1 for n, d in fast.items())
    assert {1, 2, 3, 5, 8} <= {len(c[0]) for c in CASES.values()}
    gen = {n: d for n, d in dims.items() if CASES[n][3] == "generic"}
    assert any(d[2] > 256 for d in gen.values()) and any(d[2] < 8 for d in gen.values())
    assert any(d[3] % 8 and d[1] * d[3] >= MIN_ELEMS and 8 <= d[2] <= 256 for d in gen.values())
    assert any(d[1] * d[3] < MIN_ELEMS for d in gen.values())
    assert any(c[2] == "float64" for c in CASES.values())
    assert split_bond([64] * 5, [1, 32, 32, 32, 32, 1]) in (2, 3)
    assert fast_envelope([64] * 5, [1, 32, 32, 32, 32, 1], "float32")


# ---------------------------------------------------------------------------------------------- helpers
def _cores(shape, inner, dtype, seed=0, scale=True):
    """randn cores, each scaled by 1 / sqrt(its left rank) so that entries of the tensor stay O(1)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    rs = [1] + list(inner) + [1]
    return [torch.randn(rs[k], shape[k], rs[k + 1], generator=g, device="cuda", dtype=getattr(torch, dtype))
            / (math.sqrt(rs[k]) if scale else 1.0) for k in range(len(shape))]


def _ref64(cores):
    f = cores[0].double().reshape(-1, cores[0].shape[2])
    for c in cores[1:]:
        f = (f @ c.double().reshape(c.shape[0], -1)).reshape(-1, c.shape[2])
    return f.reshape([c.shape[1] for c in cores])


def _rel(a, ref):
    return float(torch.linalg.vector_norm(a.double() - ref) / torch.linalg.vector_norm(ref))


def _int_cores(shape, inner, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rs = [1] + list(inner) + [1]
    return [torch.randint(-1, 2, (rs[k], shape[k], rs[k + 1]), generator=g, device="cuda").float()
            for k in range(len(shape))]


def _old_chain(cores):
    """Tensor.torch() as it has always run: one library product per core, left to right."""
    from tntorch_b200 import ops

    f = torch.ones(1, cores[0].shape[0], dtype=cores[0].dtype, device=cores[0].device)
    for c in cores:
        f = ops.matmul(f.contiguous(), c.reshape(c.shape[0], -1)).reshape(-1, c.shape[-1])
    return f[..., 0].reshape([c.shape[1] for c in cores])


# ---------------------------------------------------------------------------------------------- (1) exactness
# ranks <= 8 and entries in {-1, 0, 1}: every partial sum is a small integer, exact in fp32 and in its TF32 hi + lo split
INT_CASES = {"fast": ((64, 32, 16, 32), [4, 8, 4]), "fast_k8_wide": ((128, 128, 64), [8, 8]),
             "generic": ((16, 9, 7, 11), [3, 2, 3])}


@gpu
@pytest.mark.parametrize("name", list(INT_CASES))
def test_exact_on_integer_cores(name):
    import tntorch_b200 as tnb

    shape, inner = INT_CASES[name]
    assert fast_envelope(shape, [1] + inner + [1], "float32") == name.startswith("fast")
    cores = _int_cores(shape, inner, 5)
    ref = _ref64(cores)
    t = tnb.Tensor(cores)
    assert torch.equal(t.torch(dtype=torch.float32).double(), ref)
    amax = float(ref.abs().max())
    print(f"integer cores {name}: max |entry| {amax:.0f}")
    for dt, lim in ((torch.bfloat16, 256), (torch.float16, 2048)):
        keep = ref.abs() <= lim   # integers up to there are exact in the 16-bit type
        got = t.torch(dtype=dt)
        assert got.dtype == dt and torch.equal(got.double()[keep], ref[keep])
        assert int(keep.sum()) > ref.numel() // 2


# ---------------------------------------------------------------------------------------------- (2), (5) accuracy
# measured on an H100 80GB HBM3: tensor-core product 1.1e-7 .. 3.8e-7, generic fp32 4.7e-8 .. 4.1e-7, fp64 1.5e-16 .. 3.8e-16
BOUND = {"float32": 1e-6, "float64": 2e-15}


@gpu
@pytest.mark.parametrize("name", list(CASES))
def test_accuracy_against_fp64_chain(name):
    import tntorch_b200 as tnb
    from tntorch_b200 import ops

    shape, inner, dtype, path, _ = CASES[name]
    cores = _cores(shape, inner, dtype, seed=len(name))
    ref = _ref64(cores)
    t = tnb.Tensor(cores)
    dt = getattr(torch, dtype)
    n0 = ops.launch_count()
    got = t.torch(dtype=dt)
    launches = ops.launch_count() - n0
    assert got.dtype == dt and list(got.shape) == list(shape)
    assert launches == expected_launches(shape, [1] + inner + [1], dtype), (name, launches)
    e = _rel(got, ref)
    old = t.torch()
    d_old = _rel(got, old.double())
    print(f"{name} [{path}] rel. error vs fp64 chain {e:.2e}; vs Tensor.torch() {d_old:.2e} (its own error {_rel(old, ref):.2e})")
    assert e <= BOUND[dtype]
    assert d_old <= (2e-6 if dtype == "float32" else 1e-13)


GOLDEN = ["gpu_randn16x3_r3", "ragged_f32", "twin_16x5_f32", "smooth_f32_r6", "cfg1_randn16x4_f64", "ragged_f64_bigrank",
          "randn64x4_r32_f32"]


@gpu
@pytest.mark.parametrize("name", GOLDEN)
def test_accuracy_on_orthonormal_gauge_tts(name):
    """The cores tn.Tensor(X, ranks_tt=r) returns for golden cases (orthonormal but for the last)."""
    import tntorch_b200 as tnb

    spec = cases.TTSVD_CASES[name]
    X = torch.as_tensor(cases.make_dense(spec)).cuda()
    t = tnb.Tensor(X, ranks_tt=spec["ranks_tt"])
    ref = _ref64(t.cores)
    got = t.torch(dtype=X.dtype)
    e, d_old = _rel(got, ref), _rel(got, t.torch().double())
    print(f"{name}: rel. error vs fp64 chain {e:.2e}; vs Tensor.torch() {d_old:.2e}")
    assert e <= BOUND[spec["dtype"]]
    assert d_old <= (2e-6 if spec["dtype"] == "float32" else 1e-13)


@gpu
def test_argumentless_torch_is_unchanged():
    """Tensor.torch() runs the chain it always ran: the same launches, the same bits."""
    import tntorch_b200 as tnb
    from tntorch_b200 import ops

    cores = _cores((16,) * 5, [32] * 4, "float32", seed=3)
    n0 = ops.launch_count()
    want = _old_chain(cores)
    n1 = ops.launch_count()
    got = tnb.Tensor(cores).torch()
    n2 = ops.launch_count()
    assert n2 - n1 == n1 - n0 == len(cores)
    assert torch.equal(got, want)


# ---------------------------------------------------------------------------------------------- (3) 16-bit output
@gpu
@pytest.mark.parametrize("name", ["fast_k32_5d", "fast_k50_padded", "fast_k256", "generic_ragged_nc", "generic_tiny",
                                  "single_n1"])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_16bit_output_is_the_fp32_result_rounded_once(name, dt):
    import tntorch_b200 as tnb

    shape, inner, dtype, _, _ = CASES[name]
    t = tnb.Tensor(_cores(shape, inner, dtype, seed=7))
    f32 = t.torch(dtype=torch.float32)
    assert torch.equal(t.torch(dtype=dt), f32.to(dt))


@gpu
@pytest.mark.parametrize("name", ["fast_k32_5d", "generic_ragged_nc"])
def test_fp16_overflow_gives_inf_like_torch(name):
    import tntorch_b200 as tnb

    shape, inner, dtype, _, _ = CASES[name]
    cores = _cores(shape, inner, dtype, seed=9)
    cores[0] = cores[0] * 3e4   # entries O(3e4): some beyond fp16's 65504
    t = tnb.Tensor(cores)
    f32 = t.torch(dtype=torch.float32)
    h = t.torch(dtype=torch.float16)
    assert torch.equal(h, f32.to(torch.float16))
    assert bool(torch.isinf(h).any()) and not bool(torch.isinf(f32).any())


# ---------------------------------------------------------------------------------------------- (4) round trip
@gpu
@pytest.mark.parametrize("name", ["gpu_randn16x3_r3", "twin_16x5_f32", "ragged_f32"])
def test_bf16_round_trip(name):
    import tntorch_b200 as tnb
    from tntorch_b200 import ops

    spec = cases.TTSVD_CASES[name]
    Xb = torch.as_tensor(cases.make_dense(spec)).float().cuda().to(torch.bfloat16)
    t = tnb.Tensor(Xb, ranks_tt=max(Xb.shape) ** (Xb.dim() // 2))   # no truncation
    back = t.torch(dtype=torch.bfloat16)
    assert back.dtype == torch.bfloat16
    assert _rel(back, Xb.double()) <= 2.0 ** -8
    e32 = _rel(t.torch(dtype=torch.float32), Xb.double())
    e_lib = ops.tt_relative_error(Xb, t.cores)
    print(f"{name}: bf16 round trip {_rel(back, Xb.double()):.2e}, fp32 error {e32:.3e}, tt_relative_error {e_lib:.3e}")
    assert abs(e32 - e_lib) <= 1e-6


@gpu
def test_bf16_round_trip_exact_on_integers():
    import tntorch_b200 as tnb

    shape, inner = INT_CASES["generic"]
    X = _ref64(_int_cores(shape, inner, 5))
    assert float(X.abs().max()) <= 256
    Xb = X.to(torch.bfloat16)
    t = tnb.Tensor(Xb, ranks_tt=[3, 2, 3])
    back = t.torch(dtype=torch.bfloat16)
    nz = Xb != 0   # a zero comes back as the fp32 rounding residue of the SVD's factors, every other entry exactly
    assert torch.equal(back[nz], Xb[nz])
    assert float(back[~nz].float().abs().max()) <= 2.0 ** -16


# ---------------------------------------------------------------------------------------------- (6) out=, streams
@gpu
@pytest.mark.parametrize("name", ["fast_k50_padded", "generic_ragged_nc", "single_n1"])
@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16])
def test_out_buffer_and_canary(name, dt):
    import tntorch_b200 as tnb

    shape, inner, dtype, _, _ = CASES[name]
    t = tnb.Tensor(_cores(shape, inner, dtype, seed=11))
    want = t.torch(dtype=dt)
    n = want.numel()
    pad = 16 // want.element_size()
    for lead in (pad, 1):   # a 16-byte aligned buffer, and one that is not: the generic product takes it
        buf = torch.full((lead + n + 64,), 7.0, dtype=dt, device="cuda")
        out = buf[lead: lead + n].view(list(shape))
        assert (out.data_ptr() % 16 == 0) == (lead == pad)
        got = t.torch(dtype=dt, out=out)
        assert got.data_ptr() == out.data_ptr()
        if lead == pad:
            assert torch.equal(out, want)
        else:
            assert _rel(out, want.double()) <= (1e-6 if dt == torch.float32 else 2.0 ** -7)
        assert bool((buf[:lead] == 7.0).all()) and bool((buf[lead + n:] == 7.0).all())
    with pytest.raises(ValueError):
        t.torch(out=torch.empty(n + 1, dtype=want.dtype, device="cuda"))
    with pytest.raises(ValueError):
        t.torch(dtype=torch.float16, out=torch.empty(list(shape), dtype=torch.float32, device="cuda"))


@gpu
def test_two_threads_two_streams():
    import tntorch_b200 as tnb

    names = ["fast_k32_5d", "fast_k64_last_bond"]
    ts = [tnb.Tensor(_cores(*CASES[n][:3], seed=13 + i)) for i, n in enumerate(names)]
    want = [t.torch(dtype=torch.bfloat16) for t in ts]
    torch.cuda.synchronize()
    got, errs = [None, None], []

    def work(i):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for _ in range(4):
                    got[i] = ts[i].torch(dtype=torch.bfloat16)
            s.synchronize()
        except Exception as e:  # surfaced below
            errs.append(e)

    th = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errs, errs
    assert all(torch.equal(g, w) for g, w in zip(got, want))


@gpu
def test_refusals_of_the_one_call_path():
    import tntorch_b200 as tnb
    from tntorch_b200 import ops

    cp = tnb.Tensor([torch.randn(5, 3, device="cuda") for _ in range(3)])   # CP factors
    with pytest.raises(ValueError):
        cp.torch(dtype=torch.float32)
    cores = _cores((4, 5, 6), [3, 3], "float32")
    cores[1].requires_grad_(True)
    with pytest.raises(ValueError):
        tnb.Tensor(cores).torch(dtype=torch.float32)
    with pytest.raises(ValueError):
        ops.tt_decompress([torch.randn(2, 4, 3, device="cuda"), torch.randn(3, 5, 1, device="cuda")])
    with pytest.raises(NotImplementedError):
        tnb.Tensor(_cores((4, 5, 6), [3, 3], "float64")).torch(dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError):
        tnb.Tensor(_cores((4, 5, 6), [3, 3], "float32")).torch(dtype=torch.float8_e4m3fn)


@gpu
def test_tucker_factors_and_batch():
    import tntorch_b200 as tnb

    g = torch.Generator(device="cuda").manual_seed(17)
    cores = _cores((5, 6, 7), [3, 4], "float32", seed=17)
    Us = [torch.randn(9, 5, generator=g, device="cuda"), None, torch.randn(8, 7, generator=g, device="cuda")]
    t = tnb.Tensor(cores, Us=Us)
    old = t.torch()
    assert _rel(t.torch(dtype=torch.float32), old.double()) <= 2e-6
    assert torch.equal(t.torch(dtype=torch.bfloat16), t.torch(dtype=torch.float32).to(torch.bfloat16))
    X = torch.randn(3, 8, 9, 10, generator=g, device="cuda")
    tb = tnb.Tensor(X, ranks_tt=4, batch=True)
    out = torch.empty(3, 8, 9, 10, dtype=torch.float16, device="cuda")
    got = tb.torch(dtype=torch.float16, out=out)
    assert got.data_ptr() == out.data_ptr()
    assert torch.equal(out, tb.torch(dtype=torch.float32).to(torch.float16))
    assert _rel(tb.torch(dtype=torch.float32), tb.torch().double()) <= 2e-6


# ---------------------------------------------------------------------------------------------- (7) C-ABI bounds
@gpu
@pytest.mark.parametrize("name", ["fast_k50_padded", "fast_n8", "generic_k257", "generic_f64_ragged"])
def test_cabi_workspace_is_exact_and_checked(name):
    from tntorch_b200 import _lib

    shape, inner, dtype, _, _ = CASES[name]
    cores = _cores(shape, inner, dtype, seed=19)
    ranks = [1] + inner + [1]
    code = _lib.TNB_F32 if dtype == "float32" else _lib.TNB_F64
    N, L = len(shape), _lib.lib()
    sh, rk = _lib.i64(shape), _lib.i32(ranks)
    wsb = L.tnb_tt_decompress_workspace_bytes(code, code, N, sh, rk)
    assert wsb >= 256
    ws = torch.full((wsb + 4096,), 0x5A, dtype=torch.uint8, device="cuda")
    out = torch.full((math.prod(shape) + 256,), 3.0, dtype=cores[0].dtype, device="cuda")
    ptrs = (ctypes.c_void_p * N)(*[c.data_ptr() for c in cores])
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = L.tnb_tt_decompress(code, code, ptrs, N, sh, rk, ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(ws.data_ptr()),
                             wsb - 1, st)
    torch.cuda.synchronize()
    assert rc == _lib.ERR_WORKSPACE
    assert bool((out == 3.0).all()) and bool((ws == 0x5A).all())
    rc = L.tnb_tt_decompress(code, code, ptrs, N, sh, rk, ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(ws.data_ptr()),
                             wsb, st)
    torch.cuda.synchronize()
    assert rc == 0, L.tnb_last_error()
    n = math.prod(shape)
    assert bool((ws[wsb:] == 0x5A).all()) and bool((out[n:] == 3.0).all())
    assert _rel(out[:n].view(list(shape)), _ref64(cores)) <= BOUND[dtype]
    rk_bad = _lib.i32([2] + ranks[1:])
    assert L.tnb_tt_decompress(code, code, ptrs, N, sh, rk_bad, ctypes.c_void_p(out.data_ptr()),
                               ctypes.c_void_p(ws.data_ptr()), wsb, st) == _lib.ERR_INVALID
    assert L.tnb_tt_decompress(_lib.TNB_F64, _lib.TNB_BF16, ptrs, N, sh, rk, ctypes.c_void_p(out.data_ptr()),
                               ctypes.c_void_p(ws.data_ptr()), wsb, st) == _lib.ERR_UNSUPPORTED


# ---------------------------------------------------------------------------------------------- (10) TTMatrix
@gpu
@pytest.mark.parametrize("name", list(cases.TTMATRIX_CASES))
def test_ttmatrix_dtype(name):
    import tntorch_b200 as tnb

    spec = cases.TTMATRIX_CASES[name]
    M = torch.as_tensor(cases.ttmatrix_input(spec)).float().cuda()
    ttm = tnb.TTMatrix(M, ranks=spec["ranks"], input_dims=spec["input_dims"], output_dims=spec["output_dims"])
    got = ttm.torch(dtype=torch.bfloat16)
    assert got.dtype == torch.bfloat16 and got.shape == M.shape
    assert torch.equal(got, ttm.torch(dtype=torch.float32).to(torch.bfloat16))
    assert _rel(got, ttm.torch().double()) <= 2.0 ** -8


@gpu
def test_flagship_shape():
    """64^5 at rank 32, the shape the measurements are quoted for: fp32 within the bound of the chain it replaces, the
    16-bit results the fp32 one rounded."""
    import tntorch_b200 as tnb

    cores = _cores((64,) * 5, [32] * 4, "float32", seed=23)
    t = tnb.Tensor(cores)
    f32 = t.torch(dtype=torch.float32)
    old = t.torch()
    d = float(torch.linalg.vector_norm(f32 - old) / torch.linalg.vector_norm(old))
    print(f"64^5 r32: one-call fp32 vs Tensor.torch() {d:.2e}")
    assert d <= 2e-6
    del old
    for dt in (torch.bfloat16, torch.float16):
        assert torch.equal(t.torch(dtype=dt), f32.to(dt))
