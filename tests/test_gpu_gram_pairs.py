"""The K-blocked TF32 Gram runs its 128 x 256 tiles in pairs, (2j, bn) and (2j + 1, bn), in clusters of two CTAs that
share their 256-column B strip by TMA multicast (gram_tc.cuh).  CPU part: the pair enumeration and the launch it gives.
GPU part (-m gpu): G of ops.gram_kblocked against fp64, its symmetry, its repeatability and its dependence on the
reserved-SM count only through the split-K factor, at the benchmark's shape and at the pair enumeration's edge cases."""
import pytest
import torch

TC_KC, TC_MAX_SPLIT_ITERS, TN = 32, 512, 256  # gram_tc.cuh; the K-blocked mode's tiles are 256 columns wide


def _ksplit(iters, cnt, sms):
    """gram_tc.cuh gram_tc_ksplit."""
    base = max(sms // cnt if cnt < sms else 1, -(-iters // TC_MAX_SPLIT_ITERS))
    ks, best, k = base, 0.0, base
    while k <= 8 * base and k <= iters and (k == base or 64 * k <= iters):
        ctas = k * cnt
        eff = ctas / (-(-ctas // sms) * sms)
        if eff > best + 0.02:
            best, ks = eff, k
        k += 1
    return min(ks, iters)


def _kept(n):
    """The tiles (bm, bn) that touch the upper triangle, in their flat order (the partial layout's tile index)."""
    nbm, nbn = -(-n // 128), -(-n // TN)
    return [(bm, bn) for bm in range(nbm) for bn in range(nbn) if (bn + 1) * TN > bm * 128]


def _pairs(n):
    """gram_tc_kernel's cluster -> tiles: pair q is (j, bn), j-major, bn >= j; its CTAs take tile rows 2j and 2j + 1."""
    nbm, nbn = -(-n // 128), -(-n // TN)
    return [((2 * j, bn), (2 * j + 1, bn)) for j in range(-(-nbm // 2)) for bn in range(j, nbn)]


def _tile_index(n, bm, bn):
    """The kernel's flat tile id of (bm, bn): gram_tc_finalize_kernel's formula."""
    nbn = -(-n // TN)
    return sum(nbn - a * 128 // TN for a in range(bm)) + bn - bm * 128 // TN


def _ksplit_of(rows, n, sms, device_sms):
    """gram_tc_plan's split-K factor of the K-blocked Gram on `sms` usable SMs (clamped to the whole device's)."""
    iters, cnt = -(-rows // TC_KC), len(_kept(n))
    ks = _ksplit(iters, cnt, sms)
    if sms != device_sms:
        ks = min(ks, _ksplit(iters, cnt, device_sms))
    ips = -(-iters // ks)
    return -(-iters // ips)


@pytest.mark.parametrize("n", [256, 384, 512, 640, 1000, 1024, 2048, 2056, 4096])
def test_pairs_cover_the_kept_tiles(n):
    nbm = -(-n // 128)
    kept = _kept(n)
    pairs = _pairs(n)
    ctas = [t for pr in pairs for t in pr]
    real = [t for t in ctas if t[0] < nbm]
    pad = [t for t in ctas if t[0] >= nbm]
    assert sorted(real) == sorted(kept) and len(set(real)) == len(real)
    assert len(pad) == (nbm % 2), (n, pad)
    assert all(t == (nbm, nbm // 2) for t in pad)
    # both CTAs of a pair have A inside B (diagonal pair) or neither does
    for (a, b) in pairs:
        inside = [t[0] * 128 >= t[1] * TN and t[0] * 128 + 128 <= t[1] * TN + TN for t in (a, b)]
        assert inside[0] == inside[1] and inside[0] == (a[1] == a[0] // 2)
    assert [_tile_index(n, *t) for t in kept] == list(range(len(kept)))


def test_bench_shape_launch():
    """262144 x 2048 on 128 usable SMs: 36 pairs x 16 splits = 576 clusters, 9 waves of 64 pairs; the split-K factor is
    that of the 72 single tiles."""
    rows, n = 262144, 2048
    assert len(_pairs(n)) == 36 and len(_kept(n)) == 72
    ks = _ksplit_of(rows, n, 128, 132)
    assert ks == 16
    assert _ksplit(rows // TC_KC, 36, 64) == ks
    assert len(_pairs(n)) * ks == 36 * 16 and (36 * 16) % 64 == 0


def _require_tc():
    from tntorch_b200 import ops

    if not ops.has_tensorcore_path():
        pytest.fail("tensor-core path unavailable on this device (needs sm_90)")


# (rows, n): the benchmark's step-1 Gram; one diagonal pair; an odd tile-row count (a padding CTA); a partial last column
# tile with an odd tile-row count; a row count off every split boundary whose last stage ends in the first half of B
# (the second CTA's half of that stage lies past the matrix); a single split of 24 rows
SHAPES = [(262144, 2048), (40000, 256), (30000, 384), (30008, 640), (49160, 512), (24, 384)]


def _columns(n):
    """Columns whose fp64 reference is cheap and that meet every 128 x 256 tile: both ends and the middle of every
    256-column block."""
    cols = sorted({c for b in range(0, n, TN) for c in (b, b + 127, b + 128, min(b + TN, n) - 1) if c < n})
    return torch.tensor(cols)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES)
def test_gram_pairs(shape):
    from tntorch_b200 import ops

    _require_tc()
    rows, n = shape
    g = torch.Generator(device="cuda").manual_seed(31)
    A = torch.randn(rows, n, generator=g, device="cuda", dtype=torch.float32)
    B = ops.to_kblocked(A)
    dev_sms = torch.cuda.get_device_properties(0).multi_processor_count
    Gs = {}
    try:
        for r in (0, 4, 18):
            ops.set_reserved_sms(r)
            G = ops.gram_kblocked(B, rows, n)
            assert torch.equal(G, ops.gram_kblocked(B, rows, n)), r
            Gs[r] = G
    finally:
        ops.set_reserved_sms(0)
    G = Gs[0]
    assert torch.equal(G, G.T)
    cols = _columns(n).cuda()
    A64 = A.double()
    ref = A64.T @ A64[:, cols]
    scale = (A64 * A64).sum(0).max().item()
    del A64
    assert (G[:, cols] - ref).abs().max().item() / scale < 2e-3
    d = G.diagonal()[cols] / ref[cols, torch.arange(len(cols), device="cuda")]
    assert d.min().item() > 1 - 2e-3 and d.max().item() <= 1 + 1e-6
    ks = {r: _ksplit_of(rows, n, dev_sms - r, dev_sms) for r in Gs}
    for r in Gs:
        for s in Gs:
            if ks[r] == ks[s]:
                assert torch.equal(Gs[r], Gs[s]), (r, s, ks)
