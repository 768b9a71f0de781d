"""-m gpu: float16 input to the dense TT-SVD.  The fp16 tensor-core Gram (exact on integer data, noise within the level
the accept rule is given), the fp16 projection at fp32 accuracy in both output layouts and over a wide range of column
scales of V, parity of tn.Tensor / eps= / batch=True / TTMatrix on fp16-rounded golden cases against the fp64 oracle on
the same fp16 values (also scaled to fp16's subnormal and upper range), the 64^5 workload against the fp32 path on the
upcast data, and the entry points that keep rejecting fp16."""
import pytest
import torch

from gpu_util import ranks_of, relerr64
from oracle import cases
from oracle import tt_oracle as orc

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _int_f16(rows, n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(-3, 4, (rows, n), generator=g, device="cuda").to(torch.float16)


# n = 32 / 64 fold to 128 columns; 40000 + 8 rows end inside a 32-row stage; 1000 leaves a partial last tile; the
# 600000-row cases have an uneven last split-K range
@pytest.mark.parametrize("rows,n", [(40064, 32), (40064, 64), (40008, 128), (40008, 256), (20008, 1000), (12008, 2048),
                                    (600008, 64), (600008, 256)])
def test_f16_gram_exact_on_integers(rows, n):
    from tntorch_b200 import ops

    A = _int_f16(rows, n, rows + n)
    G = ops.gram_f16(A)
    Ad = A.double()
    assert torch.equal(G, Ad.T @ Ad)  # every partial sum is an integer below 2^24: exact in fp32


def _rank6_noisy(rows, n, g):
    return torch.randn(rows, 6, generator=g, device="cuda") @ torch.randn(6, n, generator=g, device="cuda") + \
        1e-3 * torch.randn(rows, n, generator=g, device="cuda")


# the two random shapes of step 0 / step 1 of 64^5 and a rank-6 signal with 1e-3 noise at the step-0 shape
@pytest.mark.parametrize("rows,n,kind", [(1 << 24, 64, "randn"), (262144, 2048, "randn"), (1 << 24, 64, "rank6")])
def test_f16_gram_noise_within_accept_level(rows, n, kind):
    """||G_f16 - (1 - c) G_fp64||_2 / ||G_fp64||_2 after the least-squares uniform shrink c stays within the level the
    accept rule is given for the fp16 Gram."""
    from tntorch_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(11)
    A = (torch.randn(rows, n, generator=g, device="cuda") if kind == "randn" else _rank6_noisy(rows, n, g)).to(torch.float16)
    G = ops.gram_f16(A)
    Gr = torch.zeros(n, n, dtype=torch.float64, device="cuda")
    for i in range(0, rows, 1 << 20):
        B = A[i: i + (1 << 20)].double()
        Gr += B.T @ B
    c = 1.0 - float((G * Gr).sum() / (Gr * Gr).sum())
    noise = float(torch.linalg.matrix_norm(G - (1 - c) * Gr, ord=2) / torch.linalg.matrix_norm(Gr, ord=2))
    print(f"fp16 Gram rows={rows} n={n} {kind}: shrink c {c:.3e}, noise {noise:.3e}")
    assert 0.0 <= c < 1e-5
    assert noise <= ops.gram_noise_level(torch.float16)


def _col_relerr(C, ref):
    """largest relative error of a column: a column whose scale of V went wrong cannot hide behind the others"""
    return float((torch.linalg.vector_norm(C.double() - ref, dim=0) / torch.linalg.vector_norm(ref, dim=0)).max())


@pytest.mark.parametrize("rows,n,r,inner", [(64 ** 4, 64, 32, 64), (131072, 64, 16, 16), (65536, 128, 48, 32),
                                            (40000, 96, 32, 0), (32768, 1024, 32, 0)])
def test_f16_projection_fp32_accuracy_and_kblocked_layout(rows, n, r, inner):
    from tntorch_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(rows + n)
    A = torch.randn(rows, n, generator=g, device="cuda").to(torch.float16)
    V = torch.randn(n, r, generator=g, device="cuda")
    Cm = ops.project_f16(A, V)
    ref = A.double() @ V.double()
    assert float(torch.linalg.vector_norm(Cm.double() - ref) / torch.linalg.vector_norm(ref)) <= 1e-6
    assert _col_relerr(Cm, ref) <= 1e-6
    if inner:
        kb = ops.project_f16(A, V, inner=inner)
        assert torch.equal(kb, ops.to_kblocked(Cm.reshape(rows // inner, inner * r)).reshape(-1))


# V's columns far below fp16's normal range (an unscaled split would lose them to subnormals), far above the unit scale,
# and both in alternate columns of one V (the scale is per column)
@pytest.mark.parametrize("scale", ["2^-20", "2^10", "mixed"])
def test_f16_projection_column_scale_range(scale):
    from tntorch_b200 import ops

    rows, n, r, inner = 131072, 64, 32, 16
    g = torch.Generator(device="cuda").manual_seed(7)
    A = torch.randn(rows, n, generator=g, device="cuda").to(torch.float16)
    V, _ = torch.linalg.qr(torch.randn(n, r, generator=g, device="cuda", dtype=torch.float64))
    V = V.float()
    if scale == "2^-20":
        V = V * 2.0 ** -20
    elif scale == "2^10":
        V = V * 2.0 ** 10
    else:
        V[:, 0::2] *= 2.0 ** -20
        V[:, 1::2] *= 2.0 ** 10
    Cm = ops.project_f16(A, V)
    ref = A.double() @ V.double()
    assert _col_relerr(Cm, ref) <= 1e-6
    kb = ops.project_f16(A, V, inner=inner)
    assert torch.equal(kb, ops.to_kblocked(Cm.reshape(rows // inner, inner * r)).reshape(-1))


def _f16_case(spec, scale=1.0):
    Xh = (torch.as_tensor(cases.make_dense(spec)).double() * scale).float().cuda().to(torch.float16)
    return Xh, Xh.double().cpu().numpy()


PARITY = [("ttsvd", k) for k in ("cfg1_randn16x4_f32", "ragged_f32", "twin_small_f32", "twin_16x5_f32", "smooth_f32_r6",
                                  "randn32x5_r32_f32", "twin32x5_r32_f32", "randn64x4_r32_f32", "eps_biggram_f32")] + \
         [("lownoise", k) for k in cases.LOWNOISE_CASES]


def _check_parity(Xh, X64, spec):
    import tntorch_b200 as tnb

    if spec.get("eps") is not None:
        t = tnb.Tensor(Xh, eps=spec["eps"])
        cores = t.decompress_tucker_factors().cores
        oc = orc.tt_svd(X64, eps=spec["eps"])
    else:
        t = tnb.Tensor(Xh, ranks_tt=spec["ranks_tt"])
        cores = t.cores
        oc = orc.tt_svd(X64, ranks_tt=spec["ranks_tt"])
    assert all(c.dtype == torch.float32 for c in cores)
    assert ranks_of(cores) == ranks_of([torch.as_tensor(c) for c in oc])
    assert abs(relerr64(X64, cores) - orc.relative_error(X64, oc)) <= TOL


@pytest.mark.parametrize("group,name", PARITY)
def test_f16_parity_with_fp64_oracle(group, name):
    spec = (cases.TTSVD_CASES if group == "ttsvd" else cases.LOWNOISE_CASES)[name]
    _check_parity(*_f16_case(spec), spec)


# randn 64^4 runs step 0 on the fp16 Gram and projection.  Scaled by 2^-20 most of its fp16 values are subnormal; by
# 2^12 the largest are near 2e4.  The relative error does not depend on the scale, so any absolute threshold in the
# sweep would show here.
@pytest.mark.parametrize("scale", [2.0 ** -20, 2.0 ** 12])
def test_f16_input_range(scale):
    spec = cases.TTSVD_CASES["randn64x4_r32_f32"]
    Xh, X64 = _f16_case(spec, scale)
    assert torch.isfinite(Xh).all()
    _check_parity(Xh, X64, spec)


def _exact_tt6_32x4(seed):
    """32^4 tensor of TT-rank 6 from cores with entries in {-1, 0, 1}: integer entries of magnitude <= 216, exact in fp16,
    so the tail a rank-6 truncation discards is zero: below the noise floor of any tensor-core Gram."""
    g = torch.Generator().manual_seed(seed)
    cores = [torch.randint(-1, 2, (r0, 32, r1), generator=g).double() for r0, r1 in ((1, 6), (6, 6), (6, 6), (6, 1))]
    X = cores[0].reshape(32, 6)
    for c in cores[1:]:
        X = (X @ c.reshape(c.shape[0], -1)).reshape(-1, c.shape[2])
    return X.reshape((32,) * 4)


def test_f16_speculation_accepted_and_rejected():
    from tntorch_b200 import ops

    # step 0 of 32^4 (32768 x 32, folded) is the only step on a tensor-core Gram: the fp16 one.  Flat random data is
    # accepted on it, on both paths; the low-noise tensor is rejected there and redone on the exact Gram, on both paths.
    g = torch.Generator(device="cuda").manual_seed(4)
    Xr = torch.randn((32,) * 4, generator=g, device="cuda").to(torch.float16)
    _, info = ops.ttsvd(Xr, rmax=6, speculate=False, return_info=True)
    assert info["tc_grams"] == 1
    _, info = ops.ttsvd(Xr, rmax=6, return_info=True)
    assert info["speculative"] == 1 and info["tc_grams"] == 1
    X64 = _exact_tt6_32x4(21)
    Xh = X64.float().cuda().to(torch.float16)
    assert torch.equal(Xh.double().cpu(), X64)
    oc = orc.tt_svd(X64.numpy(), ranks_tt=6)
    cores, info = ops.ttsvd(Xh, rmax=6, speculate=False, return_info=True)
    assert info["tc_grams"] == 0  # the fp16 Gram was rejected by the accept rule and step 0 redone exactly
    assert ranks_of(cores) == ranks_of([torch.as_tensor(c) for c in oc])
    assert abs(relerr64(X64.numpy(), cores) - orc.relative_error(X64.numpy(), oc)) <= TOL
    cores, info = ops.ttsvd(Xh, rmax=6, return_info=True)
    assert info["speculative"] == 0 and info["spec_flags"] & 1 and info["tc_grams"] == 0
    assert ranks_of(cores) == ranks_of([torch.as_tensor(c) for c in oc])
    assert abs(relerr64(X64.numpy(), cores) - orc.relative_error(X64.numpy(), oc)) <= TOL


def test_f16_batch_host_path_and_one_mode():
    import tntorch_b200 as tnb
    from tntorch_b200 import ops

    spec = cases.TTSVD_CASES["twin_16x5_f32"]
    Xh, X64 = _f16_case(spec)
    g = torch.Generator(device="cuda").manual_seed(3)
    batch = torch.stack([Xh, (Xh.float() + 0.01 * torch.randn(Xh.shape, generator=g, device="cuda")).to(torch.float16)])
    t = tnb.Tensor(batch, ranks_tt=8, batch=True)
    for b in range(2):
        cores = [c[b] for c in t.cores]
        assert all(c.dtype == torch.float32 for c in cores)
        Xb64 = batch[b].double().cpu().numpy()
        oc = orc.tt_svd(Xb64, ranks_tt=8)
        assert ranks_of(cores) == ranks_of([torch.as_tensor(c) for c in oc])
        assert abs(relerr64(Xb64, cores) - orc.relative_error(Xb64, oc)) <= TOL
    plan = ops.TTSVDPlan(list(Xh.shape), torch.float16, rmax=8, host_io=True)
    cores = plan.run_host(Xh.cpu().pin_memory())
    assert cores[0].dtype == torch.float32 and not cores[0].is_cuda
    oc = orc.tt_svd(X64, ranks_tt=8)
    assert ranks_of(cores) == ranks_of([torch.as_tensor(c) for c in oc])
    assert abs(relerr64(X64, cores) - orc.relative_error(X64, oc)) <= TOL
    one = ops.ttsvd(Xh[0, 0, 0, 0])  # N = 1: the single core is the data, converted
    assert one[0].dtype == torch.float32 and torch.equal(one[0].reshape(-1), Xh[0, 0, 0, 0].float())


def test_f16_ttmatrix():
    from tntorch_b200 import callers

    g = torch.Generator(device="cuda").manual_seed(5)
    M = torch.randn(256, 512, generator=g, device="cuda").to(torch.float16)
    tm = callers.TTMatrix(M, ranks=[8, 8], input_dims=[4, 8, 8], output_dims=[8, 8, 8])
    assert all(c.dtype == torch.float32 for c in tm.cores)
    # the fp64 oracle on the same fp16 values, viewed as the tensor with modes (i_k o_k)
    X64 = M.double().cpu().reshape(4, 8, 8, 8, 8, 8).permute(0, 3, 1, 4, 2, 5).reshape(32, 64, 64).numpy()
    oc = orc.tt_svd(X64, ranks_tt=[8, 8])
    assert [int(r) for r in tm.ranks] == [c.shape[2] for c in oc[:-1]]
    Md = M.double()
    e_h = float(torch.linalg.vector_norm(tm.torch().double() - Md) / torch.linalg.vector_norm(Md))
    assert abs(e_h - orc.relative_error(X64, oc)) <= TOL


@pytest.mark.parametrize("name", list(cases.FULL_TTSVD_CASES))
def test_f16_full_size_matches_fp32_on_upcast(name):
    from tntorch_b200 import ops

    spec = cases.FULL_TTSVD_CASES[name]
    Xh = torch.as_tensor(cases.make_dense_big(spec)).cuda().to(torch.float16)
    ch, info = ops.ttsvd(Xh, rmax=32, return_info=True)
    cf = ops.ttsvd(Xh.float(), rmax=32)
    assert ranks_of(ch) == ranks_of(cf)
    assert abs(ops.tt_relative_error(Xh, ch) - ops.tt_relative_error(Xh, cf)) <= TOL
    if spec["kind"] == "randn":
        # step 0 projected on the fp16 tensor cores and wrote the step-1 carry K-blocked
        assert info["speculative"] == 1 and info["kblocked_steps"] == 1


def test_f16_other_entry_points_still_raise():
    from tntorch_b200 import ops

    Xh = torch.randn(8, 8, 8, device="cuda").to(torch.float16)
    cores = [torch.randn(1, 8, 2, device="cuda").to(torch.float16), torch.randn(2, 8, 1, device="cuda").to(torch.float16)]
    with pytest.raises(ValueError):
        ops.tt_round(cores, rmax=1)
    with pytest.raises(ValueError):
        ops.truncated_svd(Xh[0], rmax=2)
    with pytest.raises(ValueError):
        ops.cp_als(Xh, 2)
    with pytest.raises(ValueError):  # fp16 data takes fp32 cores
        ops.tt_relative_error(Xh, [torch.randn(1, 8, 2, device="cuda"), torch.randn(2, 8, 2, device="cuda"),
                                   torch.randn(2, 8, 1, device="cuda").to(torch.float16)])
