"""-m gpu: float8 input (e4m3fn and e5m2) to the dense TT-SVD.  The fp8 tensor-core Gram (exact on integer data, on the
TMA path and on the generic path the fp8 shape check sends 16- and 48-column unfoldings to; noise within the level the
accept rule is given), the fp8 projection at fp32 accuracy in both output layouts and over a wide range of column scales
of V, parity of tn.Tensor / eps= / batch=True / TTMatrix on fp8-rounded golden cases against the fp64 oracle on the same
fp8 values (also scaled to each format's upper and subnormal range), speculation accepted and redone, the 64^5 workload
against the fp32 path on the upcast data, the host path, and the entry points that keep rejecting fp8.  fp8 tensors are
compared through .double() or .view(torch.uint8): torch has no arithmetic on them."""
import math

import pytest
import torch

from gpu_util import ranks_of, relerr64
from oracle import cases
from oracle import tt_oracle as orc

pytestmark = pytest.mark.gpu
TOL = 1e-5
F8 = [torch.float8_e4m3fn, torch.float8_e5m2]
F8_IDS = ["e4m3", "e5m2"]


def _fit(X, dt):
    """X (float) times the power of two that keeps its largest magnitude within half of the format's range: torch turns
    out-of-range e4m3fn values into NaN."""
    top = float(X.abs().max())
    half = torch.finfo(dt).max / 2
    return X if top <= half else X * 2.0 ** math.floor(math.log2(half / top))


def _int_f8(rows, n, seed, dt):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(-3, 4, (rows, n), generator=g, device="cuda").to(torch.float32).to(dt)


# n = 32 / 64 fold to 128 columns; 40000 + 8 rows end inside a 32-row stage; 1008 leaves a partial last tile; the
# 600000-row cases have an uneven last split-K range
@pytest.mark.parametrize("dt", F8, ids=F8_IDS)
@pytest.mark.parametrize("rows,n", [(40064, 32), (40064, 64), (40008, 128), (40008, 256), (20008, 1008), (12008, 2048),
                                    (600008, 64), (600008, 256)])
def test_f8_gram_exact_on_integers(rows, n, dt):
    from tntorch_b200 import ops

    A = _int_f8(rows, n, rows + n, dt)
    G = ops.gram_f8(A)
    Ad = A.double()
    assert torch.equal(G, Ad.T @ Ad)  # every partial sum is an integer below 2^24: exact in fp32


# n = 16 and 48 have no tensor-core fp8 form (the fold needs 128 % n == 0 and n >= 32): the hook refuses them and the
# sweep's step 0 takes the generic exact-product Gram.  No entry point returns that Gram for fp8 input, so it is checked
# through a truncation that only an exact Gram gets right: A has rank 6 exactly (one signed class per row times integer
# class profiles, entries in -3..3), and the rank-6 TT-SVD must reconstruct it to the fp32 rounding of its cores.  A
# Gram off by the TF32 or fp16 kernels' noise (~1e-7 .. 1e-6 of ||G||) tilts the kept subspace by about as much.
@pytest.mark.parametrize("dt", F8, ids=F8_IDS)
@pytest.mark.parametrize("n", [16, 48])
def test_f8_gram_generic_path_exact_on_integers(n, dt):
    from tntorch_b200 import ops

    A = _int_f8(4096, n, n, dt)
    with pytest.raises(NotImplementedError):
        ops.gram_f8(A)
    g = torch.Generator().manual_seed(n)
    rows = 4096
    B = torch.zeros(rows, 6, dtype=torch.float64)
    B[torch.arange(rows), torch.arange(rows) % 6] = torch.randint(0, 2, (rows,), generator=g).double() * 2 - 1
    X64 = B @ torch.randint(-3, 4, (6, n), generator=g).double()
    X8 = X64.float().cuda().to(dt)
    assert torch.equal(X8.double().cpu(), X64)
    cores, info = ops.ttsvd(X8, rmax=6, return_info=True)
    assert info["tc_grams"] == 0
    assert ranks_of(cores) == [1, 6, 1]
    assert relerr64(X64.numpy(), cores) <= 1e-6


def _rank6_noisy(rows, n, g):
    return torch.randn(rows, 6, generator=g, device="cuda") @ torch.randn(6, n, generator=g, device="cuda") + \
        1e-3 * torch.randn(rows, n, generator=g, device="cuda")


# the two random shapes of step 0 / step 1 of 64^5 and a rank-6 signal with 1e-3 noise at the step-0 shape
@pytest.mark.parametrize("dt", F8, ids=F8_IDS)
@pytest.mark.parametrize("rows,n,kind", [(1 << 24, 64, "randn"), (262144, 2048, "randn"), (1 << 24, 64, "rank6")])
def test_f8_gram_noise_within_accept_level(rows, n, kind, dt):
    """||G_f8 - (1 - c) G_fp64||_2 / ||G_fp64||_2 after the least-squares uniform shrink c stays within the level the
    accept rule is given for the fp8 Gram."""
    from tntorch_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(11)
    A = (torch.randn(rows, n, generator=g, device="cuda") if kind == "randn" else _rank6_noisy(rows, n, g)).to(dt)
    G = ops.gram_f8(A)
    Gr = torch.zeros(n, n, dtype=torch.float64, device="cuda")
    for i in range(0, rows, 1 << 20):
        B = A[i: i + (1 << 20)].double()
        Gr += B.T @ B
    c = 1.0 - float((G * Gr).sum() / (Gr * Gr).sum())
    noise = float(torch.linalg.matrix_norm(G - (1 - c) * Gr, ord=2) / torch.linalg.matrix_norm(Gr, ord=2))
    print(f"{dt} Gram rows={rows} n={n} {kind}: shrink c {c:.3e}, noise {noise:.3e}")
    assert 0.0 <= c < 1e-5
    assert noise <= ops.gram_noise_level(dt)


def _col_relerr(C, ref):
    """largest relative error of a column: a column whose scale of V went wrong cannot hide behind the others"""
    return float((torch.linalg.vector_norm(C.double() - ref, dim=0) / torch.linalg.vector_norm(ref, dim=0)).max())


# K = 64 with inner = 64 is step 0 of 64^5 (half an A box per row); K = 96 ends inside the second V box of its chunk
@pytest.mark.parametrize("dt", F8, ids=F8_IDS)
@pytest.mark.parametrize("rows,n,r,inner", [(64 ** 4, 64, 32, 64), (131072, 64, 16, 16), (65536, 128, 48, 32),
                                            (40000, 96, 32, 0), (65536, 96, 32, 16), (32768, 1024, 32, 0)])
def test_f8_projection_fp32_accuracy_and_kblocked_layout(rows, n, r, inner, dt):
    from tntorch_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(rows + n)
    A = torch.randn(rows, n, generator=g, device="cuda").to(dt)
    V = torch.randn(n, r, generator=g, device="cuda")
    Cm = ops.project_f8(A, V)
    ref = A.double() @ V.double()
    assert float(torch.linalg.vector_norm(Cm.double() - ref) / torch.linalg.vector_norm(ref)) <= 1e-6
    assert _col_relerr(Cm, ref) <= 1e-6
    if inner:
        kb = ops.project_f8(A, V, inner=inner)
        assert torch.equal(kb, ops.to_kblocked(Cm.reshape(rows // inner, inner * r)).reshape(-1))


# V's columns far below fp16's normal range (an unscaled split would lose them to subnormals), far above the unit scale,
# both in alternate columns of one V (the scale is per column), and a zero column
@pytest.mark.parametrize("dt", F8, ids=F8_IDS)
@pytest.mark.parametrize("scale", ["2^-20", "2^10", "mixed"])
def test_f8_projection_column_scale_range(scale, dt):
    from tntorch_b200 import ops

    rows, n, r, inner = 131072, 64, 32, 16
    g = torch.Generator(device="cuda").manual_seed(7)
    A = torch.randn(rows, n, generator=g, device="cuda").to(dt)
    V, _ = torch.linalg.qr(torch.randn(n, r, generator=g, device="cuda", dtype=torch.float64))
    V = V.float()
    if scale == "2^-20":
        V = V * 2.0 ** -20
    elif scale == "2^10":
        V = V * 2.0 ** 10
    else:
        V[:, 0::2] *= 2.0 ** -20
        V[:, 1::2] *= 2.0 ** 10
    V[:, 5] = 0.0
    Cm = ops.project_f8(A, V)
    ref = A.double() @ V.double()
    assert torch.equal(Cm[:, 5], torch.zeros_like(Cm[:, 5]))
    keep = [j for j in range(r) if j != 5]
    assert _col_relerr(Cm[:, keep], ref[:, keep]) <= 1e-6
    kb = ops.project_f8(A, V, inner=inner)
    assert torch.equal(kb, ops.to_kblocked(Cm.reshape(rows // inner, inner * r)).reshape(-1))


def _f8_case(spec, dt, scale=None):
    X = torch.as_tensor(cases.make_dense(spec)).double()
    X = (_fit(X, dt) if scale is None else X * scale).float().cuda()
    X8 = X.to(dt)
    return X8, X8.double().cpu().numpy()


# the fp16 list without eps_biggram_f32: rounded to fp8 (relative steps of 2^-4 and 2^-3) its discarded tail exceeds the
# eps budget at every rank up to 240, and an eps-only truncation past that rank is refused (NotImplementedError)
PARITY = [("ttsvd", k) for k in ("cfg1_randn16x4_f32", "ragged_f32", "twin_small_f32", "twin_16x5_f32", "smooth_f32_r6",
                                  "randn32x5_r32_f32", "twin32x5_r32_f32", "randn64x4_r32_f32")] + \
         [("lownoise", k) for k in cases.LOWNOISE_CASES]


def _check_parity(X8, X64, spec):
    import tntorch_b200 as tnb

    if spec.get("eps") is not None:
        t = tnb.Tensor(X8, eps=spec["eps"])
        cores = t.decompress_tucker_factors().cores
        oc = orc.tt_svd(X64, eps=spec["eps"])
    else:
        t = tnb.Tensor(X8, ranks_tt=spec["ranks_tt"])
        cores = t.cores
        oc = orc.tt_svd(X64, ranks_tt=spec["ranks_tt"])
    assert all(c.dtype == torch.float32 for c in cores)
    assert ranks_of(cores) == ranks_of([torch.as_tensor(c) for c in oc])
    assert abs(relerr64(X64, cores) - orc.relative_error(X64, oc)) <= TOL


@pytest.mark.parametrize("dt", F8, ids=F8_IDS)
@pytest.mark.parametrize("group,name", PARITY)
def test_f8_parity_with_fp64_oracle(group, name, dt):
    spec = (cases.TTSVD_CASES if group == "ttsvd" else cases.LOWNOISE_CASES)[name]
    _check_parity(*_f8_case(spec, dt), spec)


# eps-driven truncation (the tail-energy rank rule) on golden shapes, with budgets above the fp8 rounding of the data (a
# relative step of 2^-4 for e4m3, 2^-3 for e5m2): the 32^5 twin's step 0 (1048576 x 32, folded) runs on the fp8 Gram,
# the two small shapes on the generic path
EPS_PARITY = [("twin32x5_r32_f32", 0.2), ("twin32x5_r32_f32", 0.3), ("eps_twin_f64", 0.2), ("eps_smooth_f64", 0.2)]


@pytest.mark.parametrize("dt", F8, ids=F8_IDS)
@pytest.mark.parametrize("name,eps", EPS_PARITY)
def test_f8_eps_parity_with_fp64_oracle(name, eps, dt):
    """The eps-truncated TT-SVD against the oracle's on the same fp8 values (ranks and error); then tn.Tensor(X8, eps=),
    which also rounds the Tucker factors with the budget the TT-SVD left (the oracle does not model that step), must stay
    within eps of the data."""
    import tntorch_b200 as tnb
    from tntorch_b200 import ops

    spec = {k: v for k, v in cases.TTSVD_CASES[name].items() if k != "ranks_tt"}
    X8, X64 = _f8_case(spec, dt)
    cores = ops.ttsvd(X8, eps=eps)
    oc = orc.tt_svd(X64, eps=eps)
    assert all(c.dtype == torch.float32 for c in cores)
    assert ranks_of(cores) == ranks_of([torch.as_tensor(c) for c in oc])
    assert abs(relerr64(X64, cores) - orc.relative_error(X64, oc)) <= TOL
    t = tnb.Tensor(X8, eps=eps)
    assert relerr64(X64, t.decompress_tucker_factors().cores) <= eps


# randn 64^4 runs step 0 on the fp8 Gram and projection.  "top" puts its largest values just below the format's
# largest (448 for e4m3, 57344 for e5m2); "sub" scales it so that most values are subnormal in the format.  The relative
# error does not depend on the scale, so any absolute threshold in the sweep would show here.
@pytest.mark.parametrize("dt", F8, ids=F8_IDS)
@pytest.mark.parametrize("where", ["top", "sub"])
def test_f8_input_range(where, dt):
    spec = cases.TTSVD_CASES["randn64x4_r32_f32"]
    X = torch.as_tensor(cases.make_dense(spec)).double()
    fmax = torch.finfo(dt).max
    scale = 2.0 ** math.floor(math.log2(fmax / float(X.abs().max()))) if where == "top" else \
        torch.finfo(dt).smallest_normal / 4
    X8, X64 = _f8_case(spec, dt, scale)
    assert not torch.isnan(X8.double()).any()
    if where == "top":
        assert float(X8.double().abs().max()) > fmax / 2
    else:
        assert float((X8.double().abs() < torch.finfo(dt).smallest_normal).double().mean()) > 0.5
    _check_parity(X8, X64, spec)


def _exact_tt6_32x4(seed):
    """32^4 tensor of TT-rank 6 with entries in {-1, 0, 1} (exact in every fp8 format): the sum over a = 0..5 of
    outer products of four 32-vectors whose supports partition each mode, so every entry is one product of signs.  The
    tail a rank-6 truncation discards is zero: below the noise floor of any tensor-core Gram."""
    g = torch.Generator().manual_seed(seed)
    fac = []
    for _ in range(4):
        owner = torch.arange(32) % 6
        sign = torch.randint(0, 2, (32,), generator=g).double() * 2 - 1
        F = torch.zeros(32, 6, dtype=torch.float64)
        F[torch.arange(32), owner] = sign
        fac.append(F)
    return torch.einsum("ia,ja,ka,la->ijkl", *fac)


@pytest.mark.parametrize("dt", F8, ids=F8_IDS)
def test_f8_speculation_accepted_and_rejected(dt):
    from tntorch_b200 import ops

    # step 0 of 32^4 (32768 x 32, folded) is the only step on a tensor-core Gram: the fp8 one.  Flat random data is
    # accepted on it, on both paths; the exact TT-rank-6 tensor is rejected there and redone on the exact Gram, on both
    # paths.
    g = torch.Generator(device="cuda").manual_seed(4)
    Xr = torch.randn((32,) * 4, generator=g, device="cuda").to(dt)
    _, info = ops.ttsvd(Xr, rmax=6, speculate=False, return_info=True)
    assert info["tc_grams"] == 1
    _, info = ops.ttsvd(Xr, rmax=6, return_info=True)
    assert info["speculative"] == 1 and info["tc_grams"] == 1
    X64 = _exact_tt6_32x4(21)
    X8 = X64.float().cuda().to(dt)
    assert torch.equal(X8.double().cpu(), X64)
    oc = orc.tt_svd(X64.numpy(), ranks_tt=6)
    cores, info = ops.ttsvd(X8, rmax=6, speculate=False, return_info=True)
    assert info["tc_grams"] == 0  # the fp8 Gram was rejected by the accept rule and step 0 redone exactly
    assert ranks_of(cores) == ranks_of([torch.as_tensor(c) for c in oc])
    assert abs(relerr64(X64.numpy(), cores) - orc.relative_error(X64.numpy(), oc)) <= TOL
    cores, info = ops.ttsvd(X8, rmax=6, return_info=True)
    assert info["speculative"] == 0 and info["spec_flags"] & 1 and info["tc_grams"] == 0
    assert ranks_of(cores) == ranks_of([torch.as_tensor(c) for c in oc])
    assert abs(relerr64(X64.numpy(), cores) - orc.relative_error(X64.numpy(), oc)) <= TOL


@pytest.mark.parametrize("dt", F8, ids=F8_IDS)
def test_f8_accept_level_between_fp8_and_fp16(dt):
    """The host-driven sweep checks a tensor-core Gram against the level of the kernel that made it: it accepts a step
    when the discarded tail exceeds about 24 * level * lambda_0.  The exact TT-rank-6 tensor plus one entry of 0.078125
    where it is zero (exact in both formats) has a step-0 tail of about 3.8e-6 lambda_0: above the fp8 level's bound
    (6e-8 -> 1.4e-6), below the fp16 level's (3e-7 -> 7.2e-6).  So the fp8 Gram is kept, and the fp16 Gram of the same
    values is redone on the exact Gram."""
    from tntorch_b200 import ops

    X64 = _exact_tt6_32x4(21)
    assert X64[0, 1, 2, 3] == 0.0
    X64[0, 1, 2, 3] = 0.078125
    X8 = X64.float().cuda().to(dt)
    assert torch.equal(X8.double().cpu(), X64)
    oc = orc.tt_svd(X64.numpy(), ranks_tt=6)
    cores, info = ops.ttsvd(X8, rmax=6, speculate=False, return_info=True)
    assert info["tc_grams"] == 1  # accepted at the fp8 level
    assert ranks_of(cores) == ranks_of([torch.as_tensor(c) for c in oc])
    assert abs(relerr64(X64.numpy(), cores) - orc.relative_error(X64.numpy(), oc)) <= TOL
    _, info = ops.ttsvd(X8.half(), rmax=6, speculate=False, return_info=True)
    assert info["tc_grams"] == 0  # the same values as fp16: rejected at the fp16 level


@pytest.mark.parametrize("dt", F8, ids=F8_IDS)
def test_f8_batch_host_path_and_one_mode(dt):
    import tntorch_b200 as tnb
    from tntorch_b200 import ops

    spec = cases.TTSVD_CASES["twin_16x5_f32"]
    X8, X64 = _f8_case(spec, dt)
    g = torch.Generator(device="cuda").manual_seed(3)
    batch = torch.stack([X8, (X8.float() + 0.01 * torch.randn(X8.shape, generator=g, device="cuda")).to(dt)])
    t = tnb.Tensor(batch, ranks_tt=8, batch=True)
    for b in range(2):
        cores = [c[b] for c in t.cores]
        assert all(c.dtype == torch.float32 for c in cores)
        Xb64 = batch[b].double().cpu().numpy()
        oc = orc.tt_svd(Xb64, ranks_tt=8)
        assert ranks_of(cores) == ranks_of([torch.as_tensor(c) for c in oc])
        assert abs(relerr64(Xb64, cores) - orc.relative_error(Xb64, oc)) <= TOL
    plan = ops.TTSVDPlan(list(X8.shape), dt, rmax=8, host_io=True)
    cores = plan.run_host(X8.cpu().pin_memory())
    assert cores[0].dtype == torch.float32 and not cores[0].is_cuda
    oc = orc.tt_svd(X64, ranks_tt=8)
    assert ranks_of(cores) == ranks_of([torch.as_tensor(c) for c in oc])
    assert abs(relerr64(X64, cores) - orc.relative_error(X64, oc)) <= TOL
    one = ops.ttsvd(X8[0, 0, 0, 0])  # N = 1: the single core is the data, converted
    assert one[0].dtype == torch.float32 and torch.equal(one[0].reshape(-1), X8[0, 0, 0, 0].float().reshape(-1))
    t0 = tnb.Tensor(X8[0, 0, 0, 0])  # a 0-dim input becomes one mode of size 1
    assert torch.equal(t0.cores[0].reshape(-1), X8[0, 0, 0, 0].float().reshape(-1))


@pytest.mark.parametrize("dt", F8, ids=F8_IDS)
def test_f8_host_path_bitwise_equal_to_device_path(dt):
    """TTSVDPlan(host_io=True) stages the fp8 bytes (one byte per element) and runs the same sweep: the same cores."""
    from tntorch_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(9)
    X8 = torch.randn((64,) * 4, generator=g, device="cuda").to(dt)
    dev = ops.ttsvd(X8, rmax=32)
    plan = ops.TTSVDPlan(list(X8.shape), dt, rmax=32, host_io=True)
    host = plan.run_host(X8.cpu().pin_memory())
    assert len(host) == len(dev)
    for a, b in zip(host, dev):
        assert torch.equal(a, b.cpu())


@pytest.mark.parametrize("dt", F8, ids=F8_IDS)
def test_f8_ttmatrix(dt):
    from tntorch_b200 import callers

    g = torch.Generator(device="cuda").manual_seed(5)
    M = torch.randn(256, 512, generator=g, device="cuda").to(dt)
    tm = callers.TTMatrix(M, ranks=[8, 8], input_dims=[4, 8, 8], output_dims=[8, 8, 8])
    assert all(c.dtype == torch.float32 for c in tm.cores)
    # the fp64 oracle on the same fp8 values, viewed as the tensor with modes (i_k o_k)
    X64 = M.double().cpu().reshape(4, 8, 8, 8, 8, 8).permute(0, 3, 1, 4, 2, 5).reshape(32, 64, 64).numpy()
    oc = orc.tt_svd(X64, ranks_tt=[8, 8])
    assert [int(r) for r in tm.ranks] == [c.shape[2] for c in oc[:-1]]
    Md = M.double()
    e_h = float(torch.linalg.vector_norm(tm.torch().double() - Md) / torch.linalg.vector_norm(Md))
    assert abs(e_h - orc.relative_error(X64, oc)) <= TOL


@pytest.mark.parametrize("dt", F8, ids=F8_IDS)
@pytest.mark.parametrize("name", list(cases.FULL_TTSVD_CASES))
def test_f8_full_size_matches_fp32_on_upcast(name, dt):
    from tntorch_b200 import ops

    spec = cases.FULL_TTSVD_CASES[name]
    X = _fit(torch.as_tensor(cases.make_dense_big(spec)).cuda(), dt)
    X8 = X.to(dt)
    del X
    c8, info = ops.ttsvd(X8, rmax=32, return_info=True)
    cf = ops.ttsvd(X8.float(), rmax=32)
    assert ranks_of(c8) == ranks_of(cf)
    assert abs(ops.tt_relative_error(X8, c8) - ops.tt_relative_error(X8, cf)) <= TOL
    if spec["kind"] == "randn":
        # step 0 projected on the fp8 tensor cores and wrote the step-1 carry K-blocked
        assert info["speculative"] == 1 and info["kblocked_steps"] == 1


@pytest.mark.parametrize("dt", F8, ids=F8_IDS)
def test_f8_other_entry_points_still_raise(dt):
    from tntorch_b200 import ops

    X8 = torch.randn(8, 8, 8, device="cuda").to(dt)
    cores = [torch.randn(1, 8, 2, device="cuda").to(dt), torch.randn(2, 8, 1, device="cuda").to(dt)]
    with pytest.raises(ValueError):
        ops.tt_round(cores, rmax=1)
    with pytest.raises(ValueError):
        ops.truncated_svd(X8[0], rmax=2)
    with pytest.raises(ValueError):
        ops.cp_als(X8, 2)
    with pytest.raises(ValueError):  # fp8 data takes fp32 cores
        ops.tt_relative_error(X8, [torch.randn(1, 8, 2, device="cuda"), torch.randn(2, 8, 2, device="cuda"),
                                   torch.randn(2, 8, 1, device="cuda").to(dt)])


@pytest.mark.parametrize("dt", [torch.float8_e4m3fnuz, torch.float8_e5m2fnuz], ids=["e4m3fnuz", "e5m2fnuz"])
def test_f8_fnuz_formats_raise(dt):
    from tntorch_b200 import ops

    X = torch.empty(16, 16, 16, dtype=dt, device="cuda")
    with pytest.raises(ValueError):
        ops.ttsvd(X, rmax=4)
