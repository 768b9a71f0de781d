"""truncated_svd, TT sums and products and the relative-error yardstick path by path against an fp64 oracle.

Paths:
  * truncated_svd (csrc/round_impl.cuh truncated_svd_impl): the side (m <= n: Gram M M^T; m > n: M^T M), the four factor
    forms (left_ortho True / False on each side), the eigensolver eig_solve_and_rank picks by L = min(m, n) (fp64
    two-sided Jacobi below 8 and from 65 to 80, the mixed Jacobi from 8 to 64, the one-sided Jacobi from 81 to 256 with
    shared memory up to 104, ChFSI above 256 with rmax, the adaptive k = 32 -> 64 -> 128 -> 240 solve with eps only), the
    refusals, and the rank rules (rmax, eps, delta, eps + rmax, rmax > L, batch_mode).  Per case: (a) the rank (exact
    where the decision has a margin, else true rank <= r <= cap), (b) ||M - L R||^2 against the best rank-r error,
    (c) the gauge of the orthonormal factor, also at the Gram's noise floor, (d) the other factor's scaling (diag(s^2)),
    (e) the principal angle to the SVD's U_r on gapped spectra, (f) the input unchanged, (g) two calls bitwise equal;
  * tt_sum / tt_hadamard: bitwise equal to NumPy's block assembly and einsum('aib,cid->acibd') (one copy, at most one
    product and one rounding per element), at K = 1..16 operands, N = 1, 2, 6, ragged ranks and cores past 2^20 elements;
    Tensor arithmetic on Tucker and CP operands against dense fp64;
  * tt_sum_round: bitwise equal to tt_round(tt_sum(...)) on the speculative, host-driven and eps paths, and against
    oracle.round_tt of the block cores; its refusals; tn.reduce against the binary tree replayed with the oracle;
  * tt_relative_error: every data type against oracle.relative_error on exactly upcast data, the grid-striding last
    contraction, every finite fp8 code point, and its argument validation;
  * matmul (gemm_direct) at the tile edges and its N-tile refusal;
  * the callers that split at the noise floor: round_tucker, shift_mode and hadamard_sum.
The CPU part restates the truncated_svd dispatch and the sum / sum+round / relative-error sizing functions.
Run with -s to see the measured deviations."""
import ctypes as C
import operator
import zlib

import numpy as np
import pytest
import torch

from oracle import tt_oracle as orc

F32, F64 = torch.float32, torch.float64
EPS64 = float(np.finfo(np.float64).eps)

# Bounds, each at most 10x the largest value measured on an H100 SXM (132 SMs, 700 W) over the cases here; the measured
# maxima are quoted per entry (printed with -s as "MEASURED <type> <key> <value>").  A bound of 0 is a value that came out
# exactly 0 on the device.
#   tsvd_err:    (b) (||M - LR||^2 - sum_{i>=r} s_i^2) / ||M||^2          tsvd_gauge: (c) |Q^T Q - I|
#   tsvd_scale:  (d) |F^T F - diag(s_r^2)| / s_0^2                          tsvd_angle: (e) sin of the largest principal angle
#   sr_relerr:   |relerr(tt_sum_round) - relerr(oracle round_tt)|           sr_gauge:   |C C^T - I| of cores 1..N-1
#   relerr:      |tt_relative_error - oracle|                                relerr_exact: tt_relative_error of an exact TT
#   relerr_near1: the same at an error near 1                               matmul:     max |C - C64| / (|A| |B|) entrywise
#   tucker_gauge / tucker_relerr: round_tucker's |U^T U - I| and reconstruction error
#   arith:       Tensor arithmetic on TT / Tucker / CP operands, max |T - T64| / max |T64|
#   reduce / reduce_generic: tn.reduce against the replayed tree / the generic path against the fused one (relative)
#   shift_gauge / shift_relerr: shift_mode's gauge around the centre and its error against np.moveaxis (eps = 1e-6)
#   hadsum:      |hadamard_sum - exact| / (||prod|| sqrt(numel))
TOL = {
    F64: dict(tsvd_err=1.2e-15,        # 1.27e-16
              tsvd_gauge=1e-12,        # 1.02e-13
              tsvd_scale=2e-12,        # 2.03e-13
              tsvd_angle=2.7e-12,      # 2.77e-13
              sr_relerr=2.8e-13,       # 2.8e-14
              sr_gauge=1.8e-13,        # 1.85e-14
              relerr=9.9e-15,          # 9.99e-16
              relerr_exact=1.3e-15,    # 1.36e-16
              relerr_near1=0.0,        # 0
              matmul=3.8e-15,          # 3.8e-16
              tucker_gauge=7.7e-15,    # 7.77e-16
              tucker_relerr=2.2e-13,   # 2.24e-14
              arith=2.9e-15,           # 2.99e-16
              reduce=2.7e-12,          # 2.7e-13
              reduce_generic=1e-13,    # 1.07e-14
              shift_gauge=1.3e-13,     # 1.31e-14
              shift_relerr=3e-13,      # 3.09e-14
              hadsum=6.1e-15),         # 6.13e-16
    F32: dict(tsvd_err=6.5e-12,        # 6.53e-13
              tsvd_gauge=1.8e-6,       # 1.85e-7
              tsvd_scale=1.5e-4,       # 1.55e-5 (L300_adaptive_*: the fp32-block ChFSI stops at a relative 1e-6)
              tsvd_angle=9.2e-5,       # 9.22e-6
              sr_relerr=1.9e-6,        # 1.96e-7
              sr_gauge=4.8e-7,         # 4.83e-8
              relerr=1e-8,             # 1.04e-9
              relerr_exact=7e-7,       # 7.06e-8
              relerr_near1=2.2e-15,    # 2.22e-16
              matmul=2.8e-6,           # 2.89e-7
              tucker_gauge=6.8e-7,     # 6.86e-8
              tucker_relerr=2.3e-6),   # 2.34e-7
}


def bound(key, dtype, value):
    """Print a measured deviation and check it against its TOL entry."""
    print(f"\nMEASURED {str(dtype)[6:]} {key} {value:.3g}")
    tol = TOL[dtype][key]
    assert value <= tol, (key, str(dtype), value, tol)


# ==================================================================================================== dispatch
JACOBI_MAX_N = 256  # jacobi.cuh: JACOBI_MAX_N
JACOBI_SMEM_MAX_N = 104  # jacobi.cuh: JACOBI_SMEM_MAX_N
JAC2_MAX_N_F64, JAC2_MIXED_MAX_N = 80, 64  # jacobi2.cuh
GRAM_MAX_L = 46000  # sweep.cuh eig_carve: "Gram size too large"


def tsvd_side(m, n):
    """round_impl.cuh truncated_svd_impl: use_left = m <= n (the Gram M M^T), else M^T M."""
    return "left" if m <= n else "right"


def tsvd_form(m, n, left_ortho):
    """The factor truncated_svd_impl writes orthonormal, and whether the other one is built by dividing by s (the two
    forms with the gauge repair, chol_qr_repair)."""
    if m <= n:
        return ("left", False) if left_ortho else ("right", True)
    return ("left", True) if left_ortho else ("right", False)


def tsvd_eig(m, n, rmax):
    """eig_carve / eig_run / jacobi2_eigh / jacobi_eigh for the Gram of size L = min(m, n)."""
    L = min(m, n)
    if L <= JACOBI_MAX_N:  # eig_carve: L <= JACOBI_MAX_N -> the direct solver
        if L <= JAC2_MIXED_MAX_N and L >= 8:  # jacobi2_eigh: !single_precision && n <= JAC2_MIXED_MAX_N && n >= 8
            return "jac2_mixed"
        if L <= JAC2_MAX_N_F64:  # jacobi2_ok
            return "jac2_f64"
        return "onesided_smem" if L <= JACOBI_SMEM_MAX_N else "onesided_gmem"  # jacobi_eigh
    kcap = min(rmax, L) if rmax else L
    if rmax and kcap + 16 > JACOBI_MAX_N:  # eig_carve: "target rank too large for the subspace eigensolver"
        return "refused"
    if L > GRAM_MAX_L:
        return "refused"
    return "chfsi" if rmax else "adaptive"


def tsvd_adaptive_block(rank):
    """eig_solve_and_rank: k = 32, 64, 128, then 240 (JACOBI_MAX_N - 16) until the rank rule is decided; a rank above
    240 is refused."""
    for k in (32, 64, 128, 240):
        if rank < k:
            return k
    return None


# ==================================================================================================== cases
def make_matrix(m, n, spectrum, seed, rank=None):
    """fp64 matrix with the named spectrum: gauss, graded (a 1e-3 gap after `rank`), deficient (exactly rank `rank`
    as the product of two fp64 factors), zero, tiny09 / tiny11 (sigma_max 0.9e-13 / 1.1e-13)."""
    rng = np.random.default_rng(seed)
    L = min(m, n)
    if spectrum == "gauss":
        return rng.standard_normal((m, n))
    if spectrum == "zero":
        return np.zeros((m, n))
    if spectrum == "deficient":
        return rng.standard_normal((m, rank)) @ rng.standard_normal((rank, n))
    U = np.linalg.qr(rng.standard_normal((m, L)))[0]
    V = np.linalg.qr(rng.standard_normal((n, L)))[0]
    if spectrum == "graded":
        s = np.logspace(0, -2, L)
        s[rank:] *= 1e-3
    elif spectrum in ("tiny09", "tiny11"):
        s = np.linspace(1.0, 0.5, L) * (0.9e-13 if spectrum == "tiny09" else 1.1e-13)
    else:
        raise ValueError(spectrum)
    return (U * s) @ V.T


# name: (m, n, spectrum, true rank / gap position, rule kwargs, expect): expect "exact" = rank equals the oracle's with a
# margin, "bound" = the noise floor decides (true rank <= r <= cap), "zero" = the rank-1 zero split
TSVD_CASES = {
    "L5_gauss_rmax": (5, 40, "gauss", None, dict(rmax=3), "exact"),
    "L6_tall_graded_eps": (60, 6, "graded", 3, dict(eps=1e-3), "exact"),
    "L7_deficient_default": (7, 30, "deficient", 3, dict(), "bound"),
    "L10x9_deficient_eps": (10, 9, "deficient", 2, dict(eps=1e-14 / np.sqrt(3)), "bound"),
    "L9x10_deficient_eps": (9, 10, "deficient", 2, dict(eps=1e-14 / np.sqrt(3)), "bound"),
    "L32_graded_delta": (32, 200, "graded", 12, dict(delta=None), "exact"),
    "L48_tall_gauss_eps_rmax": (300, 48, "gauss", None, dict(eps=0.3, rmax=20), "exact"),
    "L64_deficient_rmax": (64, 500, "deficient", 10, dict(rmax=30, eps=0.0), "bound"),
    "L12_tall_deficient_rmax": (300, 12, "deficient", 3, dict(rmax=6, eps=0.0), "bound"),
    "L12_wide_deficient_rmax": (12, 300, "deficient", 3, dict(rmax=6, eps=0.0), "bound"),
    "L72_graded_eps": (72, 150, "graded", 20, dict(eps=1e-4), "exact"),
    "L80_tall_rmax_above_L": (400, 80, "gauss", None, dict(rmax=500), "exact"),
    "L96_graded_batch": (96, 256, "graded", 30, dict(rmax=40, batch_mode=True), "exact"),
    "L96_deficient_batch": (96, 256, "deficient", 8, dict(rmax=40, batch_mode=True), "bound"),
    "L128_tall_graded_eps": (700, 128, "graded", 50, dict(eps=1e-4), "exact"),
    "L200_deficient_default": (200, 260, "deficient", 20, dict(), "bound"),
    "L300_chfsi_rmax": (300, 900, "graded", 24, dict(rmax=24), "exact"),
    "L320_tall_chfsi_deficient": (1000, 320, "deficient", 10, dict(rmax=16, eps=0.0), "bound"),
    "L300_adaptive_k32": (300, 600, "graded", 20, dict(eps=2e-3), "exact"),
    "L300_adaptive_k64": (300, 600, "graded", 50, dict(eps=1e-3), "exact"),
    "L300_adaptive_k128": (300, 600, "graded", 100, dict(eps=1e-3), "exact"),
    "L300_adaptive_k240": (300, 600, "graded", 200, dict(eps=1e-3), "exact"),
    "L20_zero": (20, 30, "zero", None, dict(), "zero"),
    "L20_tiny09": (20, 30, "tiny09", None, dict(), "zero"),
    "L20_tiny11": (20, 30, "tiny11", None, dict(), "exact"),
}
TSVD_REFUSED = {
    "L300_rmax241": (300, 600, "gauss", None, dict(rmax=241)),
    "L300_adaptive_rank_above_240": (300, 600, "graded", 260, dict(eps=1e-3)),
}


def rule_args(kw, M):
    kw = dict(kw)
    if "delta" in kw and kw["delta"] is None:  # a delta that sits between two tail sums
        kw["delta"] = 1e-3 * float(np.linalg.norm(M)) * 0.5
    return kw


def oracle_rank(sv, kw, L, noise):
    """round.py:137-158 on the singular values sv, with the margin of the decision: the deciding tail sum's distance
    from delta^2, relative to delta^2 and in units of 1e3 x the Gram's noise (noise * sum(sv^2))."""
    lam = sv ** 2
    tr = float(lam.sum())
    cap = min(kw.get("rmax") or (1 << 30), L)
    if kw.get("batch_mode"):
        return cap, np.inf, np.inf
    if sv[0] < 1e-13:
        return 1, np.inf, np.inf
    d2 = kw["delta"] ** 2 if "delta" in kw else (kw.get("eps") or 0.0) ** 2 * tr
    tail = np.concatenate([np.cumsum(lam[::-1])[::-1], [0.0]])  # tail[r] = sum_{i >= r} lam_i
    r_rule = max(1, L - int(np.sum(tail[:L] <= d2)))
    if r_rule > cap:  # the cap decides: the rule's rank must lie above it
        gaps = [tail[cap] - d2]
    else:
        gaps = ([tail[r_rule - 1] - d2] if tail[0] > d2 else []) + ([d2 - tail[r_rule]] if r_rule < L else [])
    g = min(gaps) if gaps else np.inf
    return min(cap, r_rule), (g / d2 if d2 > 0 else np.inf), g / (1e3 * noise * tr)


def principal_sin(Q, U):
    Q = np.linalg.qr(Q)[0]
    return float(np.linalg.norm(U - Q @ (Q.T @ U), 2))


# ==================================================================================================== CPU part
def test_dispatch_restatement_reaches_every_branch():
    seen_eig, seen_form, seen_side = set(), set(), set()
    for m, n, _, _, kw, _ in TSVD_CASES.values():
        seen_eig.add(tsvd_eig(m, n, kw.get("rmax")))
        seen_side.add(tsvd_side(m, n))
        for lo in (True, False):
            seen_form.add((tsvd_side(m, n),) + tsvd_form(m, n, lo))
    for m, n, _, _, kw in TSVD_REFUSED.values():
        seen_eig.add(tsvd_eig(m, n, kw.get("rmax")))
    assert seen_eig == {"jac2_f64", "jac2_mixed", "onesided_smem", "onesided_gmem", "chfsi", "adaptive", "refused"}
    assert seen_side == {"left", "right"}
    assert len(seen_form) == 4
    # L < 8 and 65..80 both reach the fp64 two-sided Jacobi
    Ls = {min(m, n) for m, n, *_ in TSVD_CASES.values()}
    assert any(L < 8 for L in Ls) and any(65 <= L <= 80 for L in Ls)
    # the adaptive solve: one case per block size
    blocks = {tsvd_adaptive_block(g) for m, n, _, g, kw, _ in TSVD_CASES.values() if tsvd_eig(m, n, kw.get("rmax")) == "adaptive"}
    assert blocks == {32, 64, 128, 240}
    assert tsvd_adaptive_block(TSVD_REFUSED["L300_adaptive_rank_above_240"][3]) is None
    # rank rules
    rules = {tuple(sorted(k for k in kw if kw[k] is not None or k == "delta")) for *_, kw, _ in TSVD_CASES.values()}
    assert {("rmax",), ("eps",), ("delta",), ("eps", "rmax"), ("batch_mode", "rmax"), ()} <= rules
    assert any(kw.get("rmax", 0) > min(m, n) for m, n, _, _, kw, _ in TSVD_CASES.values())


def _sum_capacity(shape, ranks):
    """round_impl.cuh make_sum_dims: the summed ranks (boundaries 1) and 64-element aligned slots."""
    N = len(shape)
    rsum = [sum(r[n] for r in ranks) for n in range(N + 1)]
    rsum[0] = rsum[N] = 1
    off, slots = 0, []
    for n in range(N):
        slots.append(off)
        off += rsum[n] * shape[n] * rsum[n + 1]
        off = (off + 63) // 64 * 64
    return rsum, slots, off


@pytest.mark.parametrize("shape,ranks", [
    ((5,), [[1, 1]] * 3),
    ((7, 3), [[1, 2, 1], [1, 1, 1]]),
    ((4, 5, 6, 3, 2, 9), [[1, 3, 1, 4, 2, 5, 1], [1, 1, 1, 1, 1, 1, 1], [1, 2, 7, 2, 2, 1, 1]]),
    ((33, 17), [[1, 5, 1]] * 16),
])
def test_sum_and_sum_round_sizing(shape, ranks):
    from tntorch_b200 import _lib

    L = _lib.lib()
    N, K = len(shape), len(ranks)
    flat = [x for r in ranks for x in r]
    rsum_c, offs = (C.c_int32 * (N + 1))(), (C.c_int64 * N)()
    cap = L.tnb_tt_sum_cores_capacity(K, N, _lib.i64(list(shape)), _lib.i32(flat), rsum_c, offs)
    rsum, slots, want = _sum_capacity(shape, ranks)
    assert cap == want and list(rsum_c) == rsum and list(offs) == slots
    assert all(s % 64 == 0 for s in slots)
    rm = _lib.i32([0] * max(N - 1, 1))
    for code, esz in ((_lib.TNB_F32, 4), (_lib.TNB_F64, 8)):
        inner = L.tnb_tt_round_workspace_bytes(code, N, _lib.i64(list(shape)), _lib.i32(rsum), rm)
        got = L.tnb_tt_sum_round_workspace_bytes(code, K, N, _lib.i64(list(shape)), _lib.i32(flat), rm)
        assert inner > 0 and got == inner + (want * esz + 255) // 256 * 256 + 256
    # 17 operands and a boundary rank != 1 are refused by the sizing functions
    assert L.tnb_tt_sum_cores_capacity(17, N, _lib.i64(list(shape)), _lib.i32(flat + flat[: N + 1]), None, None) == -1
    bad = list(flat)
    bad[0] = 2
    assert L.tnb_tt_sum_cores_capacity(K, N, _lib.i64(list(shape)), _lib.i32(bad), None, None) == -1
    assert L.tnb_tt_sum_round_workspace_bytes(_lib.TNB_F32, K, N, _lib.i64(list(shape)), _lib.i32(bad), rm) == 0


def test_relative_error_sizing_and_validation():
    from tntorch_b200 import _lib

    L = _lib.lib()
    shape, ranks = [6, 1, 5, 4], [1, 3, 3, 2, 1]
    for code in (_lib.TNB_F32, _lib.TNB_F64, _lib.TNB_BF16, _lib.TNB_F16, _lib.TNB_F8E4M3, _lib.TNB_F8E5M2):
        esz = 8 if code == _lib.TNB_F64 else 4
        # acc (2 doubles) and the ping-pong F_k buffers of prod_{j<=k} I_j x r_{k+1}, k = 0..N-2 (round_impl.cuh
        # tt_relative_error_impl), each 256-byte aligned, plus 4096
        fe = [1, 1]
        rows = 1
        for k in range(len(shape) - 1):
            rows *= shape[k]
            fe[k & 1] = max(fe[k & 1], rows * ranks[k + 1])
        al = lambda b: (b + 255) // 256 * 256
        want = al(16) + al(fe[0] * esz) + al(fe[1] * esz) + 4096
        assert L.tnb_tt_relative_error_workspace_bytes(code, 4, _lib.i64(shape), _lib.i32(ranks)) == want
        for bad in ([2, 3, 3, 2, 1], [1, 3, 3, 2, 2], [1, 3, 0, 2, 1]):
            assert L.tnb_tt_relative_error_workspace_bytes(code, 4, _lib.i64(shape), _lib.i32(bad)) == 0, bad
        assert L.tnb_tt_relative_error_workspace_bytes(code, 1, _lib.i64([5]), _lib.i32([1, 1])) == 0


# ==================================================================================================== GPU part
def _run_tsvd(Md, kw, left_ortho):
    from tntorch_b200 import ops

    return ops.truncated_svd(Md, delta=kw.get("delta"), eps=kw.get("eps"), rmax=kw.get("rmax"), left_ortho=left_ortho,
                             batch_mode=kw.get("batch_mode", False), return_zero_flag=True)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("left_ortho", [True, False], ids=["lo", "ro"])
@pytest.mark.parametrize("name", list(TSVD_CASES))
def test_truncated_svd_paths(name, left_ortho, dtype):
    m, n, spectrum, g, kw, expect = TSVD_CASES[name]
    M64 = make_matrix(m, n, spectrum, seed=zlib.crc32(name.encode()) % 1000, rank=g)
    Md = torch.as_tensor(M64).to(dtype).cuda()
    M = Md.double().cpu().numpy()  # the exactly upcast input
    kw = rule_args(kw, M)
    M0 = Md.clone()
    L_, R_, zflag = _run_tsvd(Md, kw, left_ortho)
    L2, R2, _ = _run_tsvd(Md, kw, left_ortho)
    torch.cuda.synchronize()
    assert torch.equal(Md, M0)  # (f)
    assert torch.equal(L_, L2) and torch.equal(R_, R2)  # (g)
    Lh, Rh = L_.double().cpu().numpy(), R_.double().cpu().numpy()
    r = Lh.shape[1]
    assert Rh.shape == (r, n) and Lh.shape == (m, r)
    sv = np.linalg.svd(M, compute_uv=False)
    Lmin = min(m, n)
    nm2 = float(np.sum(M * M))
    if expect == "zero":
        assert r == 1 and not Lh.any() and not Rh.any()
        print(f"\n{name} {dtype} lo={left_ortho}: zero split")
        return
    eig = tsvd_eig(m, n, kw.get("rmax"))
    noise = 1e-10 if (eig in ("chfsi", "adaptive") and dtype == F32) else EPS64  # the eigensolver's resolution
    want, margin, nmargin = oracle_rank(sv, kw, Lmin, noise)
    cap = min(kw.get("rmax") or Lmin, Lmin)
    if expect == "exact":  # (a)
        assert margin >= 1e-3 and nmargin >= 1.0, (name, margin, nmargin)
        assert r == want, (r, want)
    else:  # the noise floor decides; an fp32 input carries its rounding (~1e-7 sigma_0) in every direction
        true_rank = int(np.sum(sv > (1e-10 if dtype == F64 else 1e-5) * sv[0]))
        assert min(true_rank, cap) <= r <= cap, (true_rank, r, cap)
    err = (float(np.sum((M - Lh @ Rh) ** 2)) - float(np.sum(sv[r:] ** 2))) / nm2  # (b)
    which, divides = tsvd_form(m, n, left_ortho)
    Q, F = (Lh, Rh.T) if which == "left" else (Rh.T, Lh)
    gauge = float(np.abs(Q.T @ Q - np.eye(r)).max())  # (c)
    scale = angle = None
    if sv[r - 1] > 1e-6 * sv[0]:  # (d): the kept spectrum is above the Gram's noise floor
        scale = float(np.abs(F.T @ F - np.diag(sv[:r] ** 2)).max()) / sv[0] ** 2
    if scale is not None and r < Lmin and sv[r] < 0.5 * sv[r - 1]:  # (e) gapped, kept spectrum above the floor
        U = np.linalg.svd(M, full_matrices=False)[0][:, :r]
        angle = principal_sin(Lh, U)
    print(f"\n{name} {str(dtype)[6:]} lo={left_ortho}: rank {r} (oracle {want}, margin {margin:.3g}, cap {cap}, "
          f"eig {tsvd_eig(m, n, kw.get('rmax'))}, repair form {divides}) err {err:.3g} gauge {gauge:.3g} "
          f"scale {scale if scale is None else f'{scale:.3g}'} angle {angle if angle is None else f'{angle:.3g}'}")
    bound("tsvd_err", dtype, err)
    bound("tsvd_gauge", dtype, gauge)
    if scale is not None:
        bound("tsvd_scale", dtype, scale)
    if angle is not None:
        bound("tsvd_angle", dtype, angle)
    assert bool(zflag) is False


@pytest.mark.gpu
def test_truncated_svd_batch_zero_samples():
    """batch_mode: a zero sample keeps rank min(rmax, L) with zero factors and a negative rank flag (round.py:138-142)."""
    from tntorch_b200 import ops

    Z = torch.zeros(12, 40, dtype=F64, device="cuda")
    for lo in (True, False):  # the factor that carries s (or M) is zero; the eigenvector factor may not be
        L_, R_, z = ops.truncated_svd(Z, rmax=5, left_ortho=lo, batch_mode=True, return_zero_flag=True)
        assert z and L_.shape == (12, 5) and R_.shape == (5, 40)
        assert not (R_ if lo else L_).any() and not (L_ @ R_).any()
    T = torch.zeros(40, 12, dtype=F32, device="cuda")
    for lo in (True, False):
        L_, R_, z = ops.truncated_svd(T, rmax=3, left_ortho=lo, batch_mode=True, return_zero_flag=True)
        assert z and L_.shape == (40, 3) and not (L_ @ R_).any()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(TSVD_REFUSED))
def test_truncated_svd_refusals(name):
    from tntorch_b200 import ops

    m, n, spectrum, g, kw = TSVD_REFUSED[name]
    Md = torch.as_tensor(make_matrix(m, n, spectrum, 0, g)).cuda()
    with pytest.raises((RuntimeError, NotImplementedError, ValueError), match="subspace eigensolver|rank above 240"):
        ops.truncated_svd(Md, eps=kw.get("eps"), rmax=kw.get("rmax"))


def _arena_bytes(wsb):
    """The arena size behind a sizing query's answer: tnb200.cu with_slack(b) = b + b / 8 + 4 MiB; the largest b it maps
    to at most wsb."""
    slack = lambda b: b + b // 8 + (4 << 20)
    b = (wsb - (4 << 20)) * 8 // 9
    while slack(b + 1) <= wsb:
        b += 1
    while slack(b) > wsb:
        b -= 1
    return b


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("m,n,rule", [(250, 400, dict(eps=1e-3)), (300, 256, dict(eps=1e-3)), (240, 500, dict()),
                                      (90, 100, dict(rmax=20)), (300, 900, dict(rmax=240)), (300, 900, dict(eps=1e-3))],
                         ids=["L250_eps", "L256_tall_eps", "L240_default", "L90_rmax", "L300_rmax240", "L300_eps"])
def test_truncated_svd_workspace_covers_every_request(m, n, rule, dtype):
    """tnb_truncated_svd_workspace_bytes sizes for rmax = 240; an rmax-free request up to L = 256 (the direct solver,
    whose gauge repair can keep all L vectors) must fit in the arena it sized, without the slack on top.  A short arena
    is refused before any launch."""
    from tntorch_b200 import _lib

    L = _lib.lib()
    M = torch.as_tensor(make_matrix(m, n, "graded", 1, rank=min(m, n) // 3)).to(dtype).cuda()
    code = _lib.TNB_F64 if dtype == F64 else _lib.TNB_F32
    wsb = L.tnb_truncated_svd_workspace_bytes(code, m, n)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    k = min(m, n)
    left = torch.empty(m * k, dtype=dtype, device="cuda")
    right = torch.empty(k * n, dtype=dtype, device="cuda")
    rank = (C.c_int32 * 1)()
    rc = L.tnb_truncated_svd(code, C.c_void_p(M.data_ptr()), m, n, -1.0, float(rule.get("eps", -1.0)), int(rule.get("rmax", 0)),
                             1, C.c_void_p(ws.data_ptr()), _arena_bytes(wsb), C.c_void_p(left.data_ptr()),
                             C.c_void_p(right.data_ptr()), rank, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert rc == 0, _lib.lib().tnb_last_error()
    assert 1 <= rank[0] <= k


# ------------------------------------------------------------------------------------------- sums and products
def _np_sum(ops_np, alpha, dt):
    """Block cores of sum_k alpha_k T_k: alpha_k enters the first core (rounded once from the fp64 product); N = 1 is
    the plain weighted sum of vectors, accumulated in the cores' type in operand order."""
    K, N = len(ops_np), len(ops_np[0])
    al = [1.0] * K if alpha is None else [float(a) for a in alpha]
    if N == 1:
        v = np.zeros(ops_np[0][0].shape[1], dtype=dt)
        for k in range(K):
            v = (v + (al[k] * ops_np[k][0][0, :, 0].astype(np.float64)).astype(dt)).astype(dt)
        return [v.reshape(1, -1, 1)]
    out = []
    for n in range(N):
        cs = [o[n] for o in ops_np]
        if n == 0:
            cs = [(al[k] * c.astype(np.float64)).astype(dt) for k, c in enumerate(cs)]
            out.append(np.concatenate(cs, axis=2))
        elif n == N - 1:
            out.append(np.concatenate(cs, axis=0))
        else:
            R0, R1 = sum(c.shape[0] for c in cs), sum(c.shape[2] for c in cs)
            B = np.zeros((R0, cs[0].shape[1], R1), dtype=dt)
            a = b = 0
            for c in cs:
                B[a: a + c.shape[0], :, b: b + c.shape[2]] = c
                a, b = a + c.shape[0], b + c.shape[2]
            out.append(B)
    return out


def _rand_tt_np(shape, ranks, seed):
    rng = np.random.default_rng(seed)
    rs = [1] + list(ranks) + [1]
    return [rng.standard_normal((rs[k], shape[k], rs[k + 1])) for k in range(len(shape))]


def _rand_tt(shape, ranks, seed, dtype):
    return [torch.as_tensor(c).to(dtype).cuda() for c in _rand_tt_np(shape, ranks, seed)]


SUM_CASES = {
    "N1_K3": ((37,), [[], [], []], [0.5, -1.0, 2.0]),
    "N1_K16": ((9,), [[]] * 16, None),
    "N2_K2_ragged": ((11, 7), [[3], [1]], [0.3, 0.0]),
    "N6_K3_ragged": ((4, 5, 1, 6, 3, 7), [[2, 3, 1, 4, 2], [1, 1, 1, 1, 1], [3, 1, 2, 2, 5]], [1.7, -1.0, 0.0]),
    "N6_K16": ((3, 4, 2, 3, 2, 3), [[(k % 3) + 1] * 5 for k in range(16)], [(-1) ** k * (k + 1) / 7 for k in range(16)]),
    "N3_K1": ((5, 6, 4), [[2, 3]], [-0.77]),
    "N3_big_core": ((2, 4200, 2), [[16, 16], [18, 16]], [1.0, -1.0]),  # middle core 34 * 4200 * 32 > 2^20 elements
}


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", list(SUM_CASES))
def test_tt_sum_bitwise(name, dtype):
    from tntorch_b200 import ops

    shape, ranks, alpha = SUM_CASES[name]
    ops_d = [_rand_tt(shape, rk, 100 * j + len(name), dtype) for j, rk in enumerate(ranks)]
    got = ops.tt_sum(ops_d, alpha=alpha)
    dt = np.float64 if dtype == F64 else np.float32
    want = _np_sum([[c.cpu().numpy() for c in o] for o in ops_d], alpha, dt)
    for g, w in zip(got, want):
        assert g.shape == w.shape
        assert np.array_equal(g.cpu().numpy(), w), name
    if name == "N3_big_core":
        assert got[1].numel() > 1 << 20


@pytest.mark.gpu
def test_tt_sum_refuses_17_operands():
    from tntorch_b200 import ops

    ops_d = [_rand_tt((4, 5), [2], k, F64) for k in range(17)]
    with pytest.raises(ValueError, match="between 1 and 16"):
        ops.tt_sum(ops_d)


# The library takes a train's ranks as one list r_0..r_N and reads core k as r_k x I_k x r_{k+1}.  A train whose core 0
# ends in rank 3 while core 1 starts with rank 2 has no such list: it is refused before anything launches.
UNCHAINED = {
    "tt_sum": lambda ops, a, bad: ops.tt_sum([a, bad]),
    "tt_sum_round": lambda ops, a, bad: ops.tt_sum_round([a, bad], rmax=2),
    "tt_hadamard": lambda ops, a, bad: ops.tt_hadamard(a, bad),
    "tt_hadamard_round": lambda ops, a, bad: ops.tt_hadamard_round(a, bad, rmax=2),
    "tt_round_batch": lambda ops, a, bad: ops.tt_round_batch([bad, bad], rmax=2),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(UNCHAINED))
def test_unchained_core_ranks_are_refused_before_any_launch(name):
    from tntorch_b200 import ops

    a = _rand_tt((4, 5, 6), [2, 3], 1, F64)
    bad = [torch.randn(1, 4, 3, dtype=F64, device="cuda"), torch.randn(2, 5, 3, dtype=F64, device="cuda"),
           torch.randn(3, 6, 1, dtype=F64, device="cuda")]
    before = ops.launch_count()
    with pytest.raises(ValueError, match="ranks"):
        UNCHAINED[name](ops, a, bad)
    assert ops.launch_count() == before


HAD_CASES = {
    "N1": ((13,), [], []),
    "N2_1xr_rx1": ((6, 9), [1], [4]),
    "N4_ragged": ((3, 5, 4, 6), [2, 1, 3], [3, 4, 1]),
    "N2_big_core": ((5, 20000), [8], [8]),  # core 1: 64 * 20000 > 2^20 elements
}


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", list(HAD_CASES))
def test_tt_hadamard_bitwise(name, dtype):
    from tntorch_b200 import ops

    shape, ra, rb = HAD_CASES[name]
    a, b = _rand_tt(shape, ra, 1, dtype), _rand_tt(shape, rb, 2, dtype)
    got = ops.tt_hadamard(a, b)
    for g, x, y in zip(got, a, b):
        xa, yb = x.cpu().numpy(), y.cpu().numpy()
        w = np.einsum("aib,cid->acibd", xa, yb).reshape(xa.shape[0] * yb.shape[0], xa.shape[1], -1)
        assert np.array_equal(g.cpu().numpy(), w), name
    if name == "N2_big_core":
        assert got[1].numel() > 1 << 20


def _dense(t):
    return t.torch().double().cpu().numpy()


@pytest.mark.gpu
def test_tensor_arithmetic_on_tucker_and_cp_operands():
    import tntorch_b200 as tnb

    rng = np.random.default_rng(5)
    shape = (6, 5, 7)
    tt = tnb.Tensor(_rand_tt(shape, [3, 2], 7, F64))
    Us = [torch.as_tensor(np.linalg.qr(rng.standard_normal((I, 3)))[0]).cuda() for I in shape]
    tk = tnb.Tensor(_rand_tt((3, 3, 3), [2, 2], 8, F64), Us=Us)
    cp = tnb.Tensor([torch.as_tensor(rng.standard_normal((I, 4))).cuda() for I in shape])
    A, Bk, Cc = _dense(tt), _dense(tk), _dense(cp)
    worst = 0.0
    for got, want in (((tt + tk), A + Bk), ((tk - cp), Bk - Cc), ((cp * tk), Cc * Bk), ((tk * tt), Bk * A),
                      ((cp + 1.5), Cc + 1.5), ((tk + cp), Bk + Cc)):
        worst = max(worst, float(np.abs(_dense(got) - want).max() / np.abs(want).max()))
    bound("arith", F64, worst)


# ------------------------------------------------------------------------------------------- fused sum + round
def _orc_round_of_sum(ops_d, alpha, eps, rmax):
    blocks = _np_sum([[c.double().cpu().numpy() for c in o] for o in ops_d], alpha, np.float64)
    return orc.round_tt([b.copy() for b in blocks], eps=eps, rmax=rmax)


def round_tt_margins(cores, eps, rmax, noise):
    """oracle.round_tt step by step (tensor.py:2008-2083), with each step's rank decision and its margins
    (oracle_rank): the ranks the device must reproduce where the margins are large."""
    cores = [c.copy() for c in cores]
    N = len(cores)
    rm = list(rmax) if hasattr(rmax, "__len__") else [rmax] * (N - 1)
    orc.orthogonalize_to_last(cores)
    delta = eps / max(1.0, np.sqrt(N - 1)) * float(np.linalg.norm(cores[-1]))
    out = []
    for mu in range(N - 1, 0, -1):
        c = cores[mu]
        M = c.reshape(c.shape[0], -1)
        sv = np.linalg.svd(M, compute_uv=False)
        out.append(oracle_rank(sv, dict(delta=delta, rmax=rm[mu - 1]), min(M.shape), noise))
        left, right = orc.truncated_svd(M, delta=delta, rmax=rm[mu - 1], left_ortho=False)
        cores[mu] = right.reshape(-1, c.shape[1], c.shape[2])
        cores[mu - 1] = np.einsum("ijk,kl->ijl", cores[mu - 1], left)
    return out[::-1]


SR_CASES = {
    "spec_rmax": ((8, 9, 7, 6), [[3, 4, 2], [2, 2, 2], [1, 3, 1]], [1.0, -0.5, 2.0], dict(rmax=[4, 5, 3])),
    "host_rmax": ((8, 9, 7, 6), [[3, 4, 2], [2, 2, 2], [1, 3, 1]], [1.0, -0.5, 2.0], dict(rmax=[4, 5, 3], speculate=False)),
    "eps": ((10, 9, 8, 7), [[4, 4, 4], [3, 3, 3], [2, 2, 2]], [1.0, -0.5, 2.0], dict(eps=1e-2)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", list(SR_CASES))
def test_tt_sum_round_is_round_of_sum(name, dtype):
    from tntorch_b200 import ops

    shape, ranks, alpha, kw = SR_CASES[name]
    ops_d = [_rand_tt(shape, rk, 30 + j, dtype) for j, rk in enumerate(ranks)]
    eps = kw.get("eps", 1e-14)
    spec = kw.get("speculate", True)
    fused = ops.tt_sum_round(ops_d, alpha=alpha, eps=eps, rmax=kw.get("rmax"), speculate=spec)
    plain = ops.tt_round(ops.tt_sum(ops_d, alpha=alpha), eps=eps, rmax=kw.get("rmax"), speculate=spec)
    assert [x.shape for x in fused] == [x.shape for x in plain]
    for f, p in zip(fused, plain):
        assert torch.equal(f, p), name
    oc = _orc_round_of_sum(ops_d, alpha, eps, kw.get("rmax"))
    blocks = _np_sum([[c.double().cpu().numpy() for c in o] for o in ops_d], alpha, np.float64)
    X = orc.tt_reconstruct(blocks)
    # every rank decision has a margin (an fp32 input moves the tail sums by ~1e-7 of the trace)
    steps = round_tt_margins(blocks, eps, kw.get("rmax"), EPS64 if dtype == F64 else 1e-9)
    print(f"\nsum_round {name} {str(dtype)[6:]}: oracle ranks and margins {[(r, f'{a:.3g}', f'{b:.3g}') for r, a, b in steps]}")
    assert all(a >= 1e-3 and b >= 1.0 for _, a, b in steps), steps
    assert [r for r, _, _ in steps] == [c.shape[2] for c in oc[:-1]]
    assert [c.shape[2] for c in fused] == [c.shape[2] for c in oc]
    e_dev, e_orc = orc.relative_error(X, [c.double().cpu().numpy() for c in fused]), orc.relative_error(X, oc)
    gauge = max(float(np.abs(c.reshape(c.shape[0], -1) @ c.reshape(c.shape[0], -1).T - np.eye(c.shape[0])).max())
                for c in [x.double().cpu().numpy() for x in fused[1:]])
    print(f"\nsum_round {name} {dtype}: ranks {[c.shape[2] for c in fused]} relerr {e_dev:.3g} (oracle {e_orc:.3g})")
    bound("sr_relerr", dtype, abs(e_dev - e_orc))
    bound("sr_gauge", dtype, gauge)


@pytest.mark.gpu
def test_tt_sum_round_refuses_short_buffers():
    from tntorch_b200 import _lib

    L = _lib.lib()
    shape, ranks = [6, 5, 4], [[1, 2, 3, 1], [1, 3, 2, 1]]
    ops_d = [_rand_tt(shape, r[1:-1], k, F64) for k, r in enumerate(ranks)]
    flat = [x for r in ranks for x in r]
    sh, rk, rm = _lib.i64(shape), _lib.i32(flat), _lib.i32([0, 0])
    cap = L.tnb_tt_sum_round_cores_capacity(2, 3, sh, rk, rm, None)
    wsb = L.tnb_tt_sum_round_workspace_bytes(_lib.TNB_F64, 2, 3, sh, rk, rm)
    ptrs = (C.c_void_p * 6)(*[c.data_ptr() for o in ops_d for c in o])
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    out = torch.empty(cap, dtype=F64, device="cuda")
    rks = (C.c_int32 * 4)()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    args = lambda w, c: (_lib.TNB_F64, ptrs, 2, None, 3, sh, rk, rm, 1e-14, 0, C.c_void_p(ws.data_ptr()), w,
                         C.c_void_p(out.data_ptr()), c, rks, st)
    # tnb_tt_sum_round checks the cores buffer and the whole workspace requirement (assembled cores + rounding, what
    # tnb_tt_sum_round_workspace_bytes returns) before the assembly kernels launch: one element / one byte short is refused
    out.fill_(7.0)
    assert L.tnb_tt_sum_round(*args(wsb, cap - 1)) == _lib.ERR_WORKSPACE
    assert L.tnb_tt_sum_round(*args(wsb - 1, cap)) == _lib.ERR_WORKSPACE
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())  # nothing was written
    assert L.tnb_tt_sum_round(*args(wsb, cap)) == 0
    torch.cuda.synchronize()


def _replay_reduce(tts_np, eps, rmax):
    """round.py reduce's binary tree, each node oracle.round_tt of the block cores of a + b."""
    def node(a, b):
        return orc.round_tt([c.copy() for c in _np_sum([a, b], None, np.float64)], eps=eps, rmax=rmax)

    d = {}
    for e in tts_np:
        climb = 0
        while climb in d:
            e = node(d.pop(climb), e)
            climb += 1
        d[climb] = e
    keys = list(d)
    res = d[keys[0]]
    for k in keys[1:]:
        res = node(res, d[k])
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("count", [1, 2, 3, 5, 16])
@pytest.mark.parametrize("rule", [dict(eps=1e-8), dict(rmax=3)], ids=["eps", "rmax"])
def test_reduce_matches_the_replayed_tree(count, rule):
    import tntorch_b200 as tnb
    from tntorch_b200 import ops

    shape = (7, 6, 5, 4)
    base = [_rand_tt(shape, [2, 2, 2], 50 + k, F64) for k in range(3)]
    coef = np.random.default_rng(count).standard_normal((count, 3))
    ts = [tnb.Tensor(ops.tt_sum(base, alpha=list(c))) for c in coef]
    r = tnb.reduce(ts, operator.add, **rule)
    want = _replay_reduce([[c.cpu().numpy() for c in t.cores] for t in ts], rule.get("eps", 0), rule.get("rmax"))
    got = [c.cpu().numpy() for c in r.cores]
    assert [c.shape for c in got] == [c.shape for c in want]
    X = orc.tt_reconstruct(want)
    d = float(np.linalg.norm(orc.tt_reconstruct(got) - X) / np.linalg.norm(X))
    print(f"\nreduce {count} {rule}: ranks {[c.shape[2] for c in got]}")
    bound("reduce", F64, d)
    if count > 1:  # the generic-function path (a + b, then Tensor.round: Tucker and TT rounding) agrees with the fused one
        g = tnb.reduce(ts, lambda a, b: a + b, **rule)
        bound("reduce_generic", F64, float(np.linalg.norm(_dense(g) - orc.tt_reconstruct(got)) / np.linalg.norm(X)))


# ------------------------------------------------------------------------------------------- the yardstick
RELERR_CASES = {
    "N2": ((33, 47), [5]),
    "N6_ragged_I1": ((4, 3, 1, 5, 2, 6), [2, 3, 3, 1, 4]),
    "last4096_strided": ((4100, 4096), [3]),  # 16.8M elements > 1184 * 256 threads: the grid strides
    "rows_over_2^24": ((4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 2), [2] * 13),  # 2^26 rows x 2
}
DATA_TYPES = [torch.float64, torch.float32, torch.bfloat16, torch.float16, torch.float8_e4m3fn, torch.float8_e5m2]
# every data type on the small cases and on the strided 4096-column one; the 2^27-element case on fp64, fp32 and e4m3
RELERR_RUNS = ([(nm, dt) for nm in ("N2", "N6_ragged_I1", "last4096_strided") for dt in DATA_TYPES]
               + [("rows_over_2^24", dt) for dt in (torch.float64, torch.float32, torch.float8_e4m3fn)])


@pytest.mark.gpu
@pytest.mark.parametrize("name,dtype", RELERR_RUNS, ids=[f"{nm}-{str(dt)[6:]}" for nm, dt in RELERR_RUNS])
def test_relative_error_against_oracle(name, dtype):
    from tntorch_b200 import ops

    torch.manual_seed(0)
    shape, ranks = RELERR_CASES[name]
    cdt = F64 if dtype == F64 else F32
    cores = _rand_tt(shape, ranks, 3, cdt)
    X = ops.tt_decompress([c.double() for c in cores]).to(torch.float64)
    scale = 100.0 / float(X.abs().max())  # |data| <= ~130: inside every format's finite range (e4m3 stops at 448)
    cores[0] = cores[0] * scale
    X = X * scale
    noise = torch.randn_like(X) * (0.3 * float(X.std()))
    data = (X + noise).to(dtype)
    got = ops.tt_relative_error(data, cores)
    D = data.double().cpu().numpy()
    want = orc.relative_error(D, [c.double().cpu().numpy() for c in cores])
    # an fp32 core chain rounds the reconstruction to fp32 (recon_diff_kernel: (T)s)
    print(f"\nrelerr {name} {str(dtype)[6:]}: {got:.10g} oracle {want:.10g}")
    bound("relerr", cdt, abs(got - want))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_relative_error_exact_tt_and_near_one(dtype):
    from tntorch_b200 import ops

    torch.manual_seed(1)
    cores = _rand_tt((9, 8, 7, 6), [3, 4, 2], 11, dtype)
    X = ops.tt_decompress(cores)
    bound("relerr_exact", dtype, ops.tt_relative_error(X, cores))
    Y = torch.randn_like(X)
    e1 = ops.tt_relative_error(Y, [c * 1e-3 for c in cores])
    w = orc.relative_error(Y.double().cpu().numpy(), [c.double().cpu().numpy() * 1e-3 for c in cores])
    assert abs(e1 - 1) < 0.01
    bound("relerr_near1", dtype, abs(e1 - w))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float8_e4m3fn, torch.float8_e5m2], ids=["e4m3", "e5m2"])
def test_relative_error_decodes_every_fp8_code(dtype):
    """data = every finite code point; rank-1 cores whose product is torch's decoding of those codes, exactly (fp8
    values are fp32 values and the products are by 1).  recon_diff_kernel's difference is then exactly 0 for every code
    gemm_ld decodes as torch does, and any one code decoded otherwise (zeroed, sign-flipped, scaled) makes the error
    positive.  Each binade is also checked on its own, so that a misdecode of a small code cannot hide in the sum."""
    from tntorch_b200 import ops

    codes = torch.arange(256, dtype=torch.uint8).view(dtype)
    vals = codes.float()
    fin = torch.isfinite(vals)
    codes, vals = codes[fin], vals[fin]
    exps = torch.frexp(vals)[1]
    groups = [torch.ones_like(vals, dtype=torch.bool)] + [(exps == e) & (vals != 0) for e in torch.unique(exps[vals != 0])]
    for sel in groups:
        n = int(sel.sum())
        data = codes[sel].reshape(1, n).repeat(3, 1).contiguous().cuda()
        c0 = torch.ones(1, 3, 1, device="cuda")
        c1 = vals[sel].reshape(1, n, 1).cuda()
        assert ops.tt_relative_error(data, [c0, c1]) == 0.0, vals[sel]


@pytest.mark.gpu
def test_relative_error_validates_before_launch():
    from tntorch_b200 import _lib, ops

    X = torch.randn(6, 5, 4, dtype=F64, device="cuda")
    cores = _rand_tt((6, 5, 4), [2, 3], 1, F64)
    with pytest.raises(ValueError, match="mode sizes"):
        ops.tt_relative_error(X, _rand_tt((6, 5, 5), [2, 3], 1, F64))
    with pytest.raises(ValueError, match="mode sizes"):
        ops.tt_relative_error(X, cores[:2])
    with pytest.raises(ValueError, match="ranks"):
        ops.tt_relative_error(X, [cores[0], cores[1], torch.randn(2, 4, 1, dtype=F64, device="cuda")])
    L = _lib.lib()
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    res = (C.c_double * 1)()
    ptrs = (C.c_void_p * 3)(*[c.data_ptr() for c in cores])
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for nd, rk in ((3, [2, 2, 3, 1]), (3, [1, 2, 3, 2]), (3, [1, 0, 3, 1]), (1, [1, 1])):
        rc = L.tnb_tt_relative_error(_lib.TNB_F64, C.c_void_p(X.data_ptr()), ptrs, nd, _lib.i64([6, 5, 4]), _lib.i32(rk),
                                     C.c_void_p(ws.data_ptr()), ws.numel(), res, st)
        assert rc == _lib.ERR_INVALID, (nd, rk)


# ------------------------------------------------------------------------------------------- matmul
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_matmul_tile_edges(dtype):
    from tntorch_b200 import ops

    g = torch.Generator().manual_seed(0)
    worst = 0.0
    shapes = [(M, N, K) for M in (1, 63, 64, 65) for N in (1, 63, 64, 65) for K in (1, 63, 64, 65)] + [(65, 63, 1 << 17)]
    for M, N, K in shapes:
        A = torch.randn(M, K, generator=g, dtype=F64).to(dtype)
        B = torch.randn(K, N, generator=g, dtype=F64).to(dtype)
        got = ops.matmul(A.cuda(), B.cuda()).double().cpu()
        want = A.double() @ B.double()
        scale = A.double().abs() @ B.double().abs()
        worst = max(worst, float(((got - want).abs() / scale.clamp_min(1e-300)).max()))
    bound("matmul", dtype, worst)


@pytest.mark.gpu
def test_matmul_refuses_the_n_tile_limit():
    from tntorch_b200 import ops

    N = 65536 * 64  # 65536 N tiles of 64: one past the grid's y limit
    A = torch.ones(1, 1, device="cuda")
    B = torch.ones(1, N, device="cuda")
    with pytest.raises(Exception, match="N tile count"):
        ops.matmul(A, B)


# ------------------------------------------------------------------------------------------- callers at the noise floor
def _tucker_dense(shape, mr, seed):
    """A dense tensor of multilinear rank mr (a random mr^N core times random factors): its TT, at ranks above mr,
    has a multilinear rank below its TT ranks."""
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((mr,) * len(shape))
    X = G
    for k, I in enumerate(shape):
        U = rng.standard_normal((I, mr))
        X = np.moveaxis(np.tensordot(U, np.moveaxis(X, k, 0), axes=(1, 0)), 0, k)
    return X


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_round_tucker_factors_orthonormal_at_the_noise_floor(dtype):
    import tntorch_b200 as tnb

    X = _tucker_dense((10, 9, 8, 7), 2, 4)
    t = tnb.Tensor(torch.as_tensor(X).to(dtype).cuda(), ranks_tt=4)
    cases = [("tucker_tt", t), ("t_plus_t", t + t)]
    for name, s in cases:
        ref = _dense(s)
        r = s.clone()
        r.round_tucker()
        dev = max(float(np.abs(U.double().cpu().numpy().T @ U.double().cpu().numpy() - np.eye(U.shape[1])).max())
                  for U in r.Us if U is not None)
        err = float(np.linalg.norm(_dense(r) - ref) / np.linalg.norm(ref))
        print(f"\nround_tucker {name} {dtype}: Us gauge {dev:.3g} relerr {err:.3g} ranks {[U.shape[1] for U in r.Us]}")
        bound("tucker_gauge", dtype, dev)
        bound("tucker_relerr", dtype, err)


@pytest.mark.gpu
@pytest.mark.parametrize("eps", ["same", 1e-6])
def test_shift_mode_at_the_noise_floor(eps):
    import tntorch_b200 as tnb
    from tntorch_b200 import callers

    t0 = tnb.Tensor(_rand_tt((6, 5, 7, 4, 5), [3, 4, 4, 3], 9, F64))
    s = t0 + t0
    D = _dense(s)
    callers.shift_mode(s, 1, 2, eps=eps)
    want = np.moveaxis(D, 1, 3)
    cs = [c.double().cpu().numpy() for c in s.cores]
    err = float(np.linalg.norm(orc.tt_reconstruct(cs) - want) / np.linalg.norm(want))
    # the moved mode ends at position 3 with the orthogonality centre there: cores left of it are left-orthonormal,
    # cores right of it right-orthonormal
    gl = max([float(np.abs(c.reshape(-1, c.shape[2]).T @ c.reshape(-1, c.shape[2]) - np.eye(c.shape[2])).max())
              for c in cs[:3]] + [0.0])
    gr = max([float(np.abs(c.reshape(c.shape[0], -1) @ c.reshape(c.shape[0], -1).T - np.eye(c.shape[0])).max())
              for c in cs[4:]] + [0.0])
    print(f"\nshift_mode eps={eps}: relerr {err:.3g} left gauge {gl:.3g} right gauge {gr:.3g} ranks "
          f"{[c.shape[2] for c in cs]}")
    if eps == "same":  # no rank grows; the truncation error is then whatever those ranks allow
        assert all(c.shape[2] <= 8 for c in cs)
    else:
        assert err <= 10 * eps
        bound("shift_relerr", F64, err)
    bound("shift_gauge", F64, max(gl, gr))


@pytest.mark.gpu
def test_hadamard_sum_svd_on_a_rank_deficient_running_product():
    import tntorch_b200 as tnb
    from tntorch_b200 import callers

    t = tnb.Tensor(_rand_tt((6, 5, 7, 4), [2, 3, 2], 13, F64))
    ts = [t + t, t, t * 0.5]  # the running products have multilinear rank below their Kronecker ranks
    D = _dense(ts[0]) * _dense(ts[1]) * _dense(ts[2])
    got = float(callers.hadamard_sum(ts, algorithm="svd", eps=1e-10))
    want = float(D.sum())
    scale = float(np.sqrt(np.sum(D * D)) * np.sqrt(D.size))
    print(f"\nhadamard_sum svd: {got:.12g} exact {want:.12g}")
    bound("hadsum", F64, abs(got - want) / scale)
