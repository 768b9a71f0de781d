"""-m gpu: the K-blocked carry of the speculative sweep.  The projection that writes it, the projection and the wgmma Gram
that read it, each against the row-major kernels or exact products, and the 64^5 sweep taking that path."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _require_tc():
    from tntorch_b200 import ops

    if not ops.has_tensorcore_path():
        pytest.fail("tensor-core path unavailable on this device (needs sm_90)")


# (rows, K, r, inner): the bench's step 0 (2^24 x 64 -> 32, next step I = 64); r = 16 / 48 with K not a multiple of 32
# and a row-block count that does not divide evenly among the persistent CTAs
@pytest.mark.parametrize("shape", [(2**24, 64, 32, 64), (8 * 37 * 48, 100, 16, 48), (8 * 29 * 16, 36, 48, 16),
                                   (8 * 300 * 32, 200, 32, 32)])
def test_project_kblocked_out_equals_rowmajor(shape):
    from tntorch_b200 import ops

    _require_tc()
    rows, K, r, inner = shape
    g = torch.Generator(device="cuda").manual_seed(21)
    A = torch.randn(rows, K, generator=g, device="cuda")
    V = torch.randn(K, r, generator=g, device="cuda")
    ref = ops.project(A, V, tensorcore=True)
    out = ops.project_kblocked_out(A, V, inner)
    del A
    # row a of the next step's matrix M is rows a * inner .. a * inner + inner - 1 of the product
    M = ops.from_kblocked(out, rows // inner, inner * r)
    assert torch.equal(M.reshape(rows, r), ref)


# (rows, n, r): the bench's step 1 (2^18 x 2048 -> 32); rows not a multiple of 128, n not a multiple of 32, r < 16k
@pytest.mark.parametrize("shape", [(2**18, 2048, 32), (5000, 1000, 20), (16384 + 8, 256, 64)])
def test_project_kblocked_in_equals_rowmajor(shape):
    from tntorch_b200 import ops

    _require_tc()
    rows, n, r = shape
    g = torch.Generator(device="cuda").manual_seed(22)
    A = torch.randn(rows, n, generator=g, device="cuda")
    V = torch.randn(n, r, generator=g, device="cuda")
    ref = ops.project(A, V, tensorcore=True)
    C = ops.project_kblocked_in(ops.to_kblocked(A), rows, V)
    assert torch.equal(C, ref)


# TF32-exact integer inputs: any descriptor, swizzle or slice offset error changes the result.  40000 x 2048 is split-K
# with an uneven last split; 16424 and 5000 rows end inside a 32-row stage; n = 1000 ends inside a 256-column tile.
@pytest.mark.parametrize("shape", [(40000, 2048), (16424, 256), (5000, 1000)])
def test_gram_kblocked_exact(shape):
    from tntorch_b200 import ops

    _require_tc()
    rows, n = shape
    i = torch.arange(rows, dtype=torch.float64)[:, None]
    j = torch.arange(n, dtype=torch.float64)[None, :]
    A = (((i * 7 + j * 13) % 17) - 8).float().cuda()
    G = ops.gram_kblocked(ops.to_kblocked(A), rows, n)
    assert torch.equal(G, A.double().T @ A.double())


@pytest.mark.parametrize("shape", [(40000, 2048), (5000, 1000)])
def test_gram_kblocked_matches_fp64(shape):
    from tntorch_b200 import ops

    _require_tc()
    g = torch.Generator().manual_seed(13)
    A = torch.randn(*shape, generator=g, dtype=torch.float32).cuda()
    G = ops.gram_kblocked(ops.to_kblocked(A), *shape)
    ref = A.double().T @ A.double()
    scale = ref.diagonal().max().item()
    assert (G - ref).abs().max().item() / scale < 2e-3
    assert torch.equal(G, G.T)
    d = G.diagonal() / ref.diagonal()
    assert d.min().item() > 1 - 2e-3 and d.max().item() <= 1 + 1e-6


def test_sweep_64_5_reads_a_kblocked_carry():
    """The step-0 -> step-1 carry of the 64^5 rank-32 speculative sweep is K-blocked; a 64^4 sweep has none."""
    from tntorch_b200 import ops

    _require_tc()
    g = torch.Generator(device="cuda").manual_seed(3)
    X = torch.randn(64, 64, 64, 64, 64, generator=g, device="cuda")
    cores, info = ops.ttsvd(X, rmax=32, return_info=True)
    assert info["speculative"] == 1 and info["kblocked_steps"] == 1, info
    assert [int(c.shape[2]) for c in cores] == [32, 32, 32, 32, 1]
    del X
    Y = torch.randn(64, 64, 64, 64, generator=g, device="cuda")
    _, info = ops.ttsvd(Y, rmax=32, return_info=True)
    assert info["speculative"] == 1 and info["kblocked_steps"] == 0, info
