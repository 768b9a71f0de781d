"""-m gpu: edges of the warp-specialized wgmma Gram / A^T B kernel: every wgmma width the tile planner picks besides
128 and 256 (tn = 96, 160, 224), row counts that end inside a 32-row stage or after an odd number of stages, tiles whose
A operand is not a sub-block of the B slab, and split-K over 2048 columns with an uneven last split."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _require_tc():
    from tntorch_b200 import ops

    if not ops.has_tensorcore_path():
        pytest.fail("tensor-core path unavailable on this device (needs sm_90)")


# (rows, n): tn = 96 / 160 / 224 with A outside B on the first tile row; 5013 rows end inside a stage; 40000 x 2048 is
# split-K with an uneven last split
@pytest.mark.parametrize("shape", [(6000, 96), (5013, 160), (4096 + 32, 224), (40000, 2048), (31, 96)])
def test_gram_tc_edges_match_fp64(shape):
    from tntorch_b200 import ops

    _require_tc()
    g = torch.Generator().manual_seed(13)
    A = torch.randn(*shape, generator=g, dtype=torch.float32).cuda()
    G = ops.gram(A, tensorcore=True)
    ref = A.double().T @ A.double()
    scale = ref.diagonal().max().item()
    assert (G - ref).abs().max().item() / scale < 2e-3
    assert torch.equal(G, G.T)
    d = G.diagonal() / ref.diagonal()
    assert d.min().item() > 1 - 2e-3 and d.max().item() <= 1 + 1e-6


# TF32-exact integer inputs: any descriptor, swizzle, transpose or k-permutation error changes the result
@pytest.mark.parametrize("shape", [(1000 + 3, 96), (2048 + 33, 160), (3000 + 7, 224), (16421, 2048), (31, 96)])
def test_gram_tc_edges_exact(shape):
    from tntorch_b200 import ops

    _require_tc()
    rows, n = shape
    i = torch.arange(rows, dtype=torch.float64)[:, None]
    j = torch.arange(n, dtype=torch.float64)[None, :]
    A = (((i * 7 + j * 13) % 17) - 8).float().cuda()
    G = ops.gram(A, tensorcore=True)
    assert torch.equal(G, A.double().T @ A.double())


# (K, m, n): B tiles of 96 / 160 / 224 columns, A tiles partly out of range, K not a multiple of 32
@pytest.mark.parametrize("shape", [(3001, 200, 96), (5007, 160, 160), (4096, 300, 224), (40000, 256, 2048)])
def test_atb_tc_edges_match_fp64(shape):
    from tntorch_b200 import ops

    _require_tc()
    K, m, n = shape
    g = torch.Generator().manual_seed(17)
    A = torch.randn(K, m, generator=g).cuda()
    B = torch.randn(K, n, generator=g).cuda()
    D = torch.randn(m, n, generator=g).cuda()
    C = ops.atb_tensorcore(A, B, alpha=0.5, D=D, beta=-2.0)
    ref = 0.5 * (A.double().T @ B.double()) - 2.0 * D.double()
    err = (C.double() - ref).abs().max().item() / (A.double().T @ B.double()).abs().max().item()
    assert err < 3e-3, err
    Ai = torch.randint(-8, 9, (K, m), generator=g).float().cuda()
    Bi = torch.randint(-8, 9, (K, n), generator=g).float().cuda()
    assert torch.equal(ops.atb_tensorcore(Ai, Bi).double(), Ai.double().T @ Bi.double())
