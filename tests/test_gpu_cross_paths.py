"""TT-cross path by path against an fp64 oracle (tests/cross_model.py), one sweep step at a time.

Covered, each against a plain fp64 NumPy / LAPACK statement of the same operation:
  * Householder QR (`ops.qr`, csrc/qr.cuh): tall, square, wide (rows < n), n = 1, rows = 1, shapes past the CTA's 512
    threads in both directions, a batch of different problems; Q (with LAPACK's sign convention), Q^T Q = I and
    QR = A; a zero matrix and a zero column; inputs scaled by 1e+-150 ... 1e+-300 (Q unchanged, R scaled); the refusal
    of more than 5120 columns.
  * `maxvol` (csrc/maxvol.cuh): N in {r+1, 257, 1000, 2049, 20000} x r in {1, 2, 10, 31, 64, 100} -- indices bit exact
    where the oracle's decision margins allow, C, and the swap count; exact ties in the LU pivot search and in the
    swap phase (rows duplicated with their sign flipped: the lowest index wins); max_iters = 0 and tol < 1; a batch of
    different problems equal to per-problem calls bit for bit; scaled inputs.
  * `rect_maxvol`: every branch of the parameter normalisation of `ops.rect_maxvol`, a batch whose K differ, identity
    rows at the chosen index set.
  * the index-set kernels: `cross_gather_coords` (j = 0, inner, N - 1, B > 1, ragged Is), `cross_update_lsets` /
    `_rsets` with an `active` mask (frozen rows left exactly as they were), `cross_tt_eval` (shared and per-problem
    indices, ranks 1 ... 64, N = 1 and N = 32, the refusals of rank 65, 33 modes and boundary ranks other than 1).
  * the drivers step by step: `cross` and `cross_batch` are run with `ops` wrapped so that every step's samples, Q,
    chosen rows and interpolation core are recorded; the oracle then replays the run, restarting each step from the
    device's index sets, so one early difference cannot spread.  Fixed ranks, kickrank growth, `_minimize`, `tensors=`
    with rank > 1 inputs, `function_arg="matrix"`, `record_samples`, ragged Is with Is[n] < rank, N = 2; for the batch
    ragged Is, N = 2, matrix arguments, problems converging at different sweeps (frozen ones unchanged) and rank 64.
  * scale through the whole path: cross(c f) for c = 1e-165 and 1e155 equals cross(f) with core 0 scaled by c.
  * the C ABI: null pointers and bad shapes return an error code and leave the output buffers untouched.
Index sets are compared exactly wherever the oracle's smallest decision margin exceeds MARGIN; the cases assert that it
does, so a case that turns fragile fails loudly.  Run with -s to see the measured deviations."""
import ctypes as C

import numpy as np
import pytest
import torch

import cross_model as cm

pytestmark = pytest.mark.gpu
MARGIN = 1e-9
# Sample matrices with sigma_min / sigma_max below COND have no well-determined Q (duplicate fibres from the random
# initial right sets make them exactly rank deficient).  The driver cases use seeds whose every step clears it, and
# assert so.
COND = 1e-6
# Bounds, each at most 10x the largest deviation measured on an H100 80GB HBM3 (700 W) over the cases here (printed
# with -s).  Measured:
#   qr_q |Q - Q_LAPACK| 1.0e-15; qr_orth |Q^T Q - I| 1.4e-15; qr_res |QR - A| / ||A||_2 2.3e-16;
#   qr_scale |Q(cA) - Q(A)| and |R(cA) - c R(A)| / max|c R(A)| 1.3e-15; mv_c |C - C_oracle| / max(1, max|C|) 8.0e-15;
#   rect_c 4.1e-16; eval |TT - chain| / max|chain| 4.4e-16; step_q 3.9e-13; step_core |core - oracle core| /
#   max(1, max|core|) 5.4e-13; scale_core 2.6e-14 (cross_batch of c f against f, two sweeps).
TOL = dict(qr_q=1e-14, qr_orth=1e-14, qr_res=2e-15, qr_scale=1.2e-14, mv_c=8e-14, rect_c=4e-15, eval=4e-15,
           step_q=3.9e-12, step_core=1e-12, scale_core=1.2e-13)
MEASURED = {}


def _note(key, v):
    MEASURED[key] = max(MEASURED.get(key, 0.0), float(v))
    print(f"  {key}: {float(v):.2e}")
    return float(v)


def _rel(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return float(np.abs(a - b).max() / max(1.0, np.abs(b).max())) if a.size else 0.0


def _ops():
    from tntorch_b200 import ops

    return ops


# ================================================================================================ Householder QR
QR_SHAPES = [(320, 10), (64, 64), (5, 7), (3, 40), (40, 1), (1, 6), (1, 1), (2000, 30), (700, 600), (40, 700)]


@pytest.mark.parametrize("shape", QR_SHAPES, ids=[f"{a}x{b}" for a, b in QR_SHAPES])
def test_qr_against_lapack(shape):
    ops = _ops()
    A = torch.randn(*shape, generator=torch.Generator().manual_seed(sum(shape)), dtype=torch.float64)
    Q, R = ops.qr(A.cuda(), return_r=True)
    Q, R = Q.cpu(), R.cpu()
    k = min(shape)
    Qr, Rr = torch.linalg.qr(A)
    assert Q.shape == (shape[0], k) and R.shape == (k, shape[1])
    assert _note("qr_q", (Q - Qr).abs().max()) <= TOL["qr_q"]
    assert _note("qr_orth", (Q.T @ Q - torch.eye(k, dtype=torch.float64)).abs().max()) <= TOL["qr_orth"]
    assert _note("qr_res", (Q @ R - A).abs().max() / torch.linalg.matrix_norm(A, 2)) <= TOL["qr_res"]
    assert torch.equal(torch.triu(R), R)


def test_qr_batch_of_different_problems():
    ops = _ops()
    g = torch.Generator().manual_seed(9)
    A = torch.randn(5, 300, 12, generator=g, dtype=torch.float64)
    A[1] *= 1e3
    A[2, :, 3] = A[2, :, 0]
    A[3] = torch.randn(300, 4, generator=g, dtype=torch.float64) @ torch.randn(4, 12, generator=g, dtype=torch.float64)
    Q, R = ops.qr(A.cuda(), return_r=True)
    for b in range(5):
        Q1, R1 = ops.qr(A[b].cuda(), return_r=True)
        assert torch.equal(Q[b], Q1) and torch.equal(R[b], R1)
        q = Q[b].cpu()
        assert _note("qr_orth", (q.T @ q - torch.eye(12, dtype=torch.float64)).abs().max()) <= TOL["qr_orth"]
        assert _note("qr_res", (q @ R[b].cpu() - A[b]).abs().max() / torch.linalg.matrix_norm(A[b], 2)) <= TOL["qr_res"]
    assert _note("qr_q", (Q[0].cpu() - torch.linalg.qr(A[0])[0]).abs().max()) <= TOL["qr_q"]


@pytest.mark.parametrize("shape", [(50, 6), (6, 6), (4, 9)])
def test_qr_zero_matrix_and_zero_column(shape):
    """tau = 0 for a zero column: Q completes the basis exactly like LAPACK (Q = I[:, :k] for a zero matrix)."""
    ops = _ops()
    Z = torch.zeros(*shape, dtype=torch.float64)
    Q, R = ops.qr(Z.cuda(), return_r=True)
    k = min(shape)
    assert torch.equal(Q.cpu(), torch.eye(shape[0], k, dtype=torch.float64)) and not R.abs().max()
    A = torch.randn(*shape, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    A[:, min(2, shape[1] - 1)] = 0
    Q, R = ops.qr(A.cuda(), return_r=True)
    Qr, _ = torch.linalg.qr(A)
    assert _note("qr_q", (Q.cpu() - Qr).abs().max()) <= TOL["qr_q"]
    assert _note("qr_orth", (Q.cpu().T @ Q.cpu() - torch.eye(k, dtype=torch.float64)).abs().max()) <= TOL["qr_orth"]


SCALES = [1e150, 1e-150, 1e160, 1e-160, 1e200, 1e-200, 1e300, 1e-300]


@pytest.mark.parametrize("c", SCALES, ids=[f"{c:.0e}" for c in SCALES])
@pytest.mark.parametrize("shape", [(320, 10), (10, 320)], ids=["tall", "wide"])
def test_qr_is_scale_invariant(shape, c):
    """The reflector norm is taken dlarfg-style (scaled by the column's largest |value|): an unscaled sum of squares
    underflows below ~1e-160 (tau = 0, Q = I) and overflows above ~1e154 (NaN)."""
    ops = _ops()
    A = torch.randn(*shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    Q0, R0 = ops.qr(A.cuda(), return_r=True)
    Q, R = ops.qr((c * A).cuda(), return_r=True)
    assert torch.isfinite(Q).all() and torch.isfinite(R).all()
    assert _note("qr_scale", (Q - Q0).abs().max()) <= TOL["qr_scale"]
    assert _note("qr_scale", ((R - c * R0).abs().max() / (c * R0.abs().max()))) <= TOL["qr_scale"]


def test_qr_propagates_nan():
    """A NaN below the diagonal, alongside zeros only, still reaches Q and R: the column's max reduction keeps NaN."""
    ops = _ops()
    A = torch.randn(40, 5, generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    A[1:, 0] = 0.0
    A[17, 0] = float("nan")
    Q, R = ops.qr(A.cuda(), return_r=True)
    assert torch.isnan(Q).any() and torch.isnan(R).any()


def test_qr_refuses_more_than_5120_columns():
    ops = _ops()
    with pytest.raises(NotImplementedError):
        ops.qr(torch.zeros(5121, 5121, dtype=torch.float64, device="cuda"))


# ================================================================================================ maxvol
MV_N = [None, 257, 1000, 2049, 20000]  # None: r + 1
MV_R = [1, 2, 10, 31, 64, 100]
MV_CASES = [(n if n is not None else r + 1, r) for n in MV_N for r in MV_R if n is None or n > r]


def _mv_input(N, r, seed):
    return np.random.default_rng(seed).standard_normal((N, r))


@pytest.mark.parametrize("N,r", MV_CASES, ids=[f"{n}x{r}" for n, r in MV_CASES])
def test_maxvol_against_oracle(N, r):
    ops = _ops()
    A = _mv_input(N, r, 1000 * r + N)
    oi, oC, info = cm.maxvol(A)
    assert info["margin"] > MARGIN, info["margin"]
    idx, Cd, iters = ops.maxvol(torch.as_tensor(A).cuda(), return_iters=True)
    assert idx.cpu().tolist() == list(oi)
    assert iters == [info["iters"]]
    assert _note("mv_c", _rel(Cd.cpu().numpy(), oC)) <= TOL["mv_c"]


def test_maxvol_exact_ties_lowest_index_wins():
    """Rows duplicated with their sign flipped tie exactly (the LU updates and solves of a and -a are exact negations):
    the lowest index wins, in the LU pivot search (LAPACK idamax) and in the swap phase (NumPy argmax over r x N)."""
    ops = _ops()
    base = _mv_input(200, 6, 77)
    piv, _ = cm._lu_pivots(base)
    oi0, _, info0 = cm.maxvol(base)
    swapped_in = [int(j) for j in oi0 if int(j) not in set(piv.tolist())]
    assert swapped_in and info0["iters"] > 0
    # the first LU pivot and a row the swap phase brings in, each duplicated at the end with the sign flipped
    A = np.vstack([base, -base[piv[0]], -base[swapped_in[0]]])
    oi, oC, info = cm.maxvol(A)
    assert info["lu"][0] == 0.0 and 0.0 in info["swap"]  # both ties are met
    idx, Cd, iters = ops.maxvol(torch.as_tensor(A).cuda(), return_iters=True)
    assert idx.cpu().tolist() == list(oi) and 200 not in oi and 201 not in oi and swapped_in[0] in oi
    assert iters == [info["iters"]]
    assert _note("mv_c", _rel(Cd.cpu().numpy(), oC)) <= TOL["mv_c"]


def test_maxvol_stopping_rules():
    ops = _ops()
    A = _mv_input(500, 8, 3)
    idx0, _, it0 = ops.maxvol(torch.as_tensor(A).cuda(), max_iters=0, return_iters=True)
    piv, lu = cm._lu_pivots(A)
    assert min(lu) > MARGIN and idx0.cpu().tolist() == list(piv) and it0 == [0]
    # tol < 1 is clamped to 1 (maxvol.py:122-123).  At tol = 1 the final stop test meets |C| = 1 on the identity rows,
    # a decision at the rounding level (margin 0), so the two tolerances are compared with each other, bit for bit
    r1 = ops.maxvol(torch.as_tensor(A).cuda(), tol=1.0, return_iters=True)
    r05 = ops.maxvol(torch.as_tensor(A).cuda(), tol=0.5, return_iters=True)
    assert torch.equal(r1[0], r05[0]) and torch.equal(r1[1], r05[1]) and r1[2] == r05[2]
    oi1, _, info1 = cm.maxvol(A, max_iters=1)
    assert info1["margin"] > MARGIN and info1["iters"] == 1 and cm.maxvol(A)[2]["iters"] > 1
    idx1, _, it1 = ops.maxvol(torch.as_tensor(A).cuda(), max_iters=1, return_iters=True)
    assert idx1.cpu().tolist() == list(oi1) and it1 == [1]


def test_maxvol_batch_equals_single_calls():
    ops = _ops()
    rng = np.random.default_rng(11)
    A = np.stack([rng.standard_normal((700, 12)) * s for s in (1.0, 1e-3, 7.0, 1.0)])
    A[3] = np.linalg.qr(A[3])[0]
    idx, Cd, iters = ops.maxvol(torch.as_tensor(A).cuda(), return_iters=True)
    for b in range(4):
        i1, C1, it1 = ops.maxvol(torch.as_tensor(A[b]).cuda(), return_iters=True)
        assert torch.equal(idx[b], i1) and torch.equal(Cd[b], C1) and iters[b] == it1[0]
        oi, _, info = cm.maxvol(A[b])
        assert info["margin"] > MARGIN and idx[b].cpu().tolist() == list(oi)


@pytest.mark.parametrize("c", [1e-150, 1e150, 1e-300, 1e300], ids=["1e-150", "1e150", "1e-300", "1e300"])
def test_maxvol_scaled_input(c):
    ops = _ops()
    A = _mv_input(1000, 10, 5)
    i0, C0 = ops.maxvol(torch.as_tensor(A).cuda())
    i1, C1 = ops.maxvol(torch.as_tensor(c * A).cuda())
    assert torch.equal(i0, i1)
    assert _note("mv_c", _rel(C1.cpu().numpy(), C0.cpu().numpy())) <= TOL["mv_c"]


# ================================================================================================ rect_maxvol
# (N, r, tol, maxK, minK, min_add_K, start_maxvol_iters): every branch of the normalisation (maxvol.py:54-66)
RECT_CASES = {
    "defaults": (300, 8, 1.0, None, None, None, 10),
    "maxK_gt_N": (60, 6, 0.2, 500, None, None, 10),
    "maxK_lt_r": (300, 8, 1.0, 3, None, None, 10),
    "minK_gt_N": (40, 5, 5.0, None, 100, None, 10),
    "minK_gt_maxK": (300, 8, 1.0, 12, 20, None, 10),
    "min_add_K": (300, 8, 5.0, 30, None, 6, 10),
    "start_iters_0": (300, 8, 1.0, None, None, None, 0),
    "tol_large": (300, 8, 100.0, None, None, None, 10),
}


@pytest.mark.parametrize("name", list(RECT_CASES))
def test_rect_maxvol_parameters(name):
    ops = _ops()
    N, r, tol, maxK, minK, add, it = RECT_CASES[name]
    A = _mv_input(N, r, 300 + N + r)
    kw = dict(tol=tol, maxK=maxK, minK=minK, min_add_K=add, start_maxvol_iters=it)
    oi, oC, info = cm.rect_maxvol(A, **kw)
    assert info["margin"] > MARGIN, info["margin"]
    idx, Cd = ops.rect_maxvol(torch.as_tensor(A).cuda(), **kw)
    assert idx.cpu().tolist() == list(oi)
    Cd = Cd.cpu().numpy()
    assert _note("rect_c", _rel(Cd, oC)) <= TOL["rect_c"]
    assert np.array_equal(Cd[idx.cpu().numpy()], np.eye(len(oi)))  # identity_submatrix=True


def test_rect_maxvol_batch_with_different_K():
    ops = _ops()
    rng = np.random.default_rng(21)
    A = np.stack([rng.standard_normal((200, 6)), np.linalg.qr(rng.standard_normal((200, 6)))[0], rng.standard_normal((200, 6))])
    A[2, :, 5] *= 1e-2
    outs = ops.rect_maxvol(torch.as_tensor(A).cuda(), tol=1.0, maxK=40)
    Ks = []
    for b in range(3):
        oi, oC, info = cm.rect_maxvol(A[b], tol=1.0, maxK=40)
        assert info["margin"] > MARGIN
        assert outs[b][0].cpu().tolist() == list(oi)
        assert _note("rect_c", _rel(outs[b][1].cpu().numpy(), oC)) <= TOL["rect_c"]
        Ks.append(len(oi))
    assert len(set(Ks)) > 1, Ks


# ================================================================================================ index-set kernels
def _ragged_grid(Is, seed):
    rng = np.random.default_rng(seed)
    axes = [rng.standard_normal(I) for I in Is]
    grid = np.zeros((len(Is), max(Is)))
    for k, a in enumerate(axes):
        grid[k, : len(a)] = a
    return axes, grid


@pytest.mark.parametrize("j", [0, 2, 4])
def test_cross_gather_coords(j):
    ops = _ops()
    Is = [3, 7, 5, 9, 4]
    N, B, Rl, Rr = 5, 3, 2 if j else 1, 3 if j < 4 else 1
    axes, grid = _ragged_grid(Is, j)
    rng = np.random.default_rng(40 + j)
    ls = np.stack([rng.integers(0, Is[k], (B, Rl)) for k in range(j)], axis=2) if j else np.zeros((B, 1, 0), int)
    rs = np.stack([rng.integers(0, Is[k], (B, Rr)) for k in range(j + 1, N)], axis=2) if j < N - 1 else np.zeros((B, 1, 0), int)
    X = ops.cross_gather_coords(torch.as_tensor(ls, dtype=torch.int32).cuda(), torch.as_tensor(rs, dtype=torch.int32).cuda(),
                                torch.as_tensor(grid).cuda(), N, j, Is[j])
    for b in range(B):
        lset = np.c_[np.zeros(Rl, int), ls[b]]
        rset = np.c_[rs[b], np.zeros(Rr, int)]
        M = cm.fibres(lset, rset, Is[j])
        P = M.shape[0]
        for k in range(N):
            assert np.array_equal(X[k][b * P: (b + 1) * P].cpu().numpy(), axes[k][M[:, k]])


def test_cross_update_sets_with_frozen_problems():
    ops = _ops()
    rng = np.random.default_rng(50)
    B, Rl, I, Rn, j = 4, 3, 5, 4, 2
    ls = rng.integers(0, 9, (B, Rl, j)).astype(np.int32)
    local = np.stack([rng.choice(Rl * I, Rn, replace=False) for _ in range(B)]).astype(np.int32)
    active = torch.tensor([1, 0, 1, 0], dtype=torch.int32, device="cuda")
    sentinel = torch.full((B, Rn, j + 1), -7, dtype=torch.int32, device="cuda")
    out = ops.cross_update_lsets(torch.as_tensor(ls).cuda(), torch.as_tensor(local).cuda(), I, active, sentinel.clone())
    for b in range(B):
        if active[b]:
            lr, li = np.divmod(local[b], I)
            assert np.array_equal(out[b].cpu().numpy(), np.c_[ls[b][lr], li])
        else:
            assert (out[b] == -7).all()
    fresh = ops.cross_update_lsets(torch.as_tensor(ls).cuda(), torch.as_tensor(local).cuda(), I)
    assert torch.equal(fresh[0], out[0]) and torch.equal(fresh[2], out[2])
    # right sets: local indexes (i, c) of the (I * Rr) x Rp matrix
    Rr, Rp, ln = 3, 4, 2
    rs = rng.integers(0, 9, (B, Rr, ln)).astype(np.int32)
    local = np.stack([rng.choice(I * Rr, Rp, replace=False) for _ in range(B)]).astype(np.int32)
    sentinel = torch.full((B, Rp, ln + 1), -9, dtype=torch.int32, device="cuda")
    out = ops.cross_update_rsets(torch.as_tensor(rs).cuda(), torch.as_tensor(local).cuda(), Rr, active, sentinel.clone())
    for b in range(B):
        if active[b]:
            li, lr = np.divmod(local[b], Rr)
            assert np.array_equal(out[b].cpu().numpy(), np.c_[li, rs[b][lr]])
        else:
            assert (out[b] == -9).all()


def _chain(cores, idx):
    """[B, P] values of B TTs (cores [B, r, I, r']) at idx [P, N] or [B, P, N], in fp64 on the host."""
    B = cores[0].shape[0]
    out = []
    for b in range(B):
        M = idx[b] if idx.ndim == 3 else idx
        out.append(cm.tt_values([c[b] for c in cores], M))
    return np.stack(out)


@pytest.mark.parametrize("N,rank", [(1, 1), (2, 64), (4, 17), (6, 1), (32, 3), (3, 64)])
def test_cross_tt_eval(N, rank):
    ops = _ops()
    rng = np.random.default_rng(N * 100 + rank)
    Is = [int(rng.integers(2, 9)) for _ in range(N)]
    Rs = [1] + [rank] * (N - 1) + [1]
    B, P = 3, 57
    cores = [rng.standard_normal((B, Rs[n], Is[n], Rs[n + 1])) / np.sqrt(Rs[n]) for n in range(N)]
    dc = [torch.as_tensor(c).cuda() for c in cores]
    shared = np.stack([rng.integers(0, I, P) for I in Is], axis=1).astype(np.int32)
    per = np.stack([np.stack([rng.integers(0, I, P) for I in Is], axis=1) for _ in range(B)]).astype(np.int32)
    for idx in (shared, per):
        got = ops.cross_tt_eval(dc, torch.as_tensor(idx).cuda()).cpu().numpy()
        ref = _chain(cores, idx)
        assert _note("eval", np.abs(got - ref).max() / np.abs(ref).max()) <= TOL["eval"]


def test_cross_tt_eval_refusals():
    ops = _ops()
    idx = torch.zeros(4, 3, dtype=torch.int32, device="cuda")
    ok = [torch.ones(1, 1, 2, 2, dtype=torch.float64, device="cuda"), torch.ones(1, 2, 2, 2, dtype=torch.float64, device="cuda"),
          torch.ones(1, 2, 2, 1, dtype=torch.float64, device="cuda")]
    ops.cross_tt_eval(ok, idx)
    big = [torch.ones(1, 1, 2, 65, dtype=torch.float64, device="cuda"), torch.ones(1, 65, 2, 1, dtype=torch.float64, device="cuda")]
    with pytest.raises(NotImplementedError):
        ops.cross_tt_eval(big, idx[:, :2])
    many = [torch.ones(1, 1, 2, 1, dtype=torch.float64, device="cuda")] * 33
    with pytest.raises(ValueError):
        ops.cross_tt_eval(many, torch.zeros(4, 33, dtype=torch.int32, device="cuda"))
    with pytest.raises(ValueError):  # boundary ranks must be 1
        ops.cross_tt_eval([torch.ones(1, 2, 2, 2, dtype=torch.float64, device="cuda")] * 3, idx)


# ================================================================================================ drivers, step by step
class Recorder:
    """Wraps the ops the drivers call and records every call's inputs and outputs (on the host)."""

    def __init__(self, monkeypatch):
        ops = _ops()
        self.calls = []
        for name in ("qr", "maxvol", "rect_maxvol", "cross_update_lsets", "cross_update_rsets", "cross_gather_coords"):
            real = getattr(ops, name)
            monkeypatch.setattr(ops, name, self._wrap(name, real))

    def _wrap(self, name, real):
        def f(*a, **k):
            out = real(*a, **k)
            host = lambda x: x.detach().cpu().clone() if isinstance(x, torch.Tensor) else x  # noqa: E731
            self.calls.append((name, [host(x) for x in a], tuple(host(x) for x in out) if isinstance(out, tuple) else host(out)))
            return out
        return f

    def of(self, *names):
        return [c for c in self.calls if c[0] in names]


def _replay_cross(prob, rec, fcalls, info, kw, seed, exact_coords=True):
    """Replays a recorded tn.cross run with the oracle, each step restarted from the device's index sets."""
    steps = rec.of("qr")
    picks = rec.of("maxvol", "rect_maxvol")
    assert len(steps) == len(picks)
    evals = fcalls[1:]  # fcalls[0]: the validation set
    pos = {"s": 0, "e": 0}
    dev = {"q": 0.0, "core": 0.0}

    def on_step(kind, j, s, sets):
        e = evals[pos["e"]]
        pos["e"] += 1
        for x, y in zip(e[0], s.xs):
            if exact_coords:
                assert np.array_equal(x, y)
            else:
                assert np.abs(x - y).max() <= 1e-13 * max(1.0, np.abs(y).max())
        if kind == "F":
            return None
        q_in, Qd = steps[pos["s"]][1][0].numpy(), steps[pos["s"]][2]
        Qd = Qd.numpy() if isinstance(Qd, torch.Tensor) else Qd[0].numpy()
        local_d, Cd = picks[pos["s"]][2][0].numpy(), picks[pos["s"]][2][1].numpy()
        pos["s"] += 1
        assert np.abs(q_in - (s.V if kind == "L" else s.V.T)).max() <= 1e-14 * np.abs(s.V).max()
        dev["q"] = max(dev["q"], np.abs(Qd - s.Q).max())
        assert s.margin > MARGIN and s.cond > COND, (kind, j, s.margin, s.cond)
        assert list(local_d) == list(s.local), (kind, j)
        core_d = Cd.reshape(s.core.shape) if kind == "L" else Cd.T.reshape(s.core.shape)
        dev["core"] = max(dev["core"], _rel(core_d, s.core))
        lset, rset = sets[0][j], sets[1][j]
        if kind == "L":
            lr, li = np.divmod(local_d.astype(np.int64), prob.Is[j])
            return np.c_[lset[lr], li]
        li, lr = np.divmod(local_d.astype(np.int64), s.core.shape[2])
        return np.c_[li, rset[lr]]

    np.random.seed(seed)
    torch.manual_seed(seed)
    cores, oinfo = cm.run(prob, on_step=on_step, **kw)
    assert pos["s"] == len(steps) and pos["e"] == len(evals)
    assert _note("step_q", dev["q"]) <= TOL["step_q"]
    assert _note("step_core", dev["core"]) <= TOL["step_core"]
    assert list(info["Rs"]) == list(oinfo["Rs"]) and int(info["nsamples"]) == oinfo["nsamples"]
    for a, b in zip(info["lsets"], oinfo["lsets"]):
        assert np.array_equal(a, b)
    for a, b in zip(info["rsets"], oinfo["rsets"]):
        assert np.array_equal(a, b)
    return cores, oinfo


def _wavy(lib):
    def f(*xs):
        s = 0.3 + 0 * xs[0]
        for k, x in enumerate(xs):
            s = s + (k + 1.3) * x + 0.7 * x * xs[k - 1]
        return lib.sin(3.1 * s) + 1.5 * lib.cos(s * s) + 2.5
    return f


def _random_axes(Is, seed):
    rng = np.random.default_rng(seed)
    return [rng.uniform(-1.0, 1.0, I) for I in Is]


CROSS_DRIVER_CASES = {
    "fixed_ranks": dict(seed=2, Is=[9, 8, 10, 7], kw=dict(ranks_tt=3, max_iter=3, eps=0.0)),
    "kickrank": dict(seed=1, Is=[8, 9, 7, 8], kw=dict(kickrank=2, rmax=5, max_iter=4, eps=1e-14)),
    "minimize": dict(seed=8, Is=[10, 9, 8], kw=dict(ranks_tt=3, max_iter=3, eps=0.0), minimize=True),
    "matrix_arg": dict(seed=1, Is=[7, 9, 8], kw=dict(ranks_tt=4, max_iter=2, eps=0.0), matrix=True),
    "record_samples": dict(seed=1, Is=[9, 8, 7], kw=dict(ranks_tt=3, max_iter=2, eps=0.0), record=True),
    "ragged_small_modes": dict(seed=3, Is=[3, 11, 2, 9, 4], kw=dict(ranks_tt=5, max_iter=2, eps=0.0)),
    "two_modes": dict(seed=3, Is=[13, 11], kw=dict(ranks_tt=4, max_iter=3, eps=0.0)),
    "tensors_rank3": dict(seed=2, Is=[7, 8, 6, 9], kw=dict(ranks_tt=3, max_iter=2, eps=0.0), tensors=True),
}


@pytest.mark.parametrize("name", list(CROSS_DRIVER_CASES))
def test_cross_step_by_step(name, monkeypatch):
    import tntorch_b200 as tnb

    spec = CROSS_DRIVER_CASES[name]
    Is, kw, seed = spec["Is"], dict(spec["kw"]), spec["seed"]
    fcalls = []
    ftorch, fnp = _wavy(torch), _wavy(np)
    if spec.get("tensors"):
        rng = np.random.default_rng(seed)
        tts = []
        for t in range(2):
            Rs = [1] + [3] * (len(Is) - 1) + [1]
            tts.append([rng.standard_normal((Rs[n], Is[n], Rs[n + 1])) / 2 for n in range(len(Is))])
        prob = cm.Problem(lambda a, b: fnp(a, b), tensors=tts)
        fdev = lambda a, b: ftorch(a, b)  # noqa: E731
        dev_kw = dict(tensors=[tnb.Tensor([torch.as_tensor(c).cuda() for c in t]) for t in tts])
    else:
        axes = _random_axes(Is, seed)
        if spec.get("matrix"):
            prob = cm.Problem(lambda X: fnp(*X.T), domain=axes, function_arg="matrix")
            fdev = lambda X: ftorch(*X.T)  # noqa: E731
            dev_kw = dict(domain=[torch.as_tensor(a) for a in axes], function_arg="matrix")
        else:
            prob = cm.Problem(fnp, domain=axes, minimize=bool(spec.get("minimize")))
            fdev = ftorch
            dev_kw = dict(domain=[torch.as_tensor(a) for a in axes])

    def traced(*args):
        y = fdev(*args)
        xs = [a.cpu().numpy() for a in (args[0].T if spec.get("matrix") else args)]
        fcalls.append((xs, y.detach().cpu().numpy()))
        return y

    rec = Recorder(monkeypatch)
    np.random.seed(seed)
    torch.manual_seed(seed)
    t, info = tnb.cross(traced, verbose=False, return_info=True, suppress_warnings=True,
                        record_samples=bool(spec.get("record")), _minimize=bool(spec.get("minimize")), **dev_kw, **kw)
    cores, oinfo = _replay_cross(prob, rec, fcalls, info, kw, seed, exact_coords=not spec.get("tensors"))
    if spec.get("minimize"):
        assert abs(float(info["min"]) - float(oinfo["min"])) <= 1e-14 and tuple(info["argmin"]) == oinfo["argmin"]
    if spec.get("record"):
        pos = np.concatenate([np.stack(x, axis=1) for x, _ in fcalls[1:]])
        vals = np.concatenate([y for _, y in fcalls[1:]])
        assert np.array_equal(info["sample_positions"].cpu().numpy(), pos)
        assert np.array_equal(info["sample_values"].cpu().numpy(), vals)
    if name == "kickrank":
        assert max(oinfo["Rs"]) == 5 and len(oinfo["val_epss"]) == 4
    if name == "ragged_small_modes":
        assert list(oinfo["Rs"]) == [1, 3, 5, 5, 4, 1]
    for n, c in enumerate(t.cores):
        assert _note("step_core", _rel(c.cpu().numpy(), cores[n])) <= TOL["step_core"]


def _batch_family(lib, kind):
    """Problem b of a family whose members converge at different sweeps with ranks 2 and eps 1e-10: sin(a_b + sum x)
    has TT rank 2 (converges in the first sweep); the wavy members never converge.  The rough members oscillate too
    fast for any low rank, so their sample matrices stay well conditioned at rank 64."""
    def make(b):
        if kind[b] == "rough":
            g = _wavy(lib)
            return lambda *xs: lib.sin(997.0 * g(*xs)) + 2.0 + 0.1 * b
        if kind[b] == "exact":
            def f(*xs):
                s = 0.25 * b + 0 * xs[0]
                for x in xs:
                    s = s + x
                return lib.sin(s)
            return f
        g = _wavy(lib)
        return lambda *xs: g(*xs) + 0.1 * b
    return make


BATCH_CASES = {
    "converge_mixed": dict(seed=2, Is=[8, 9, 7, 8], ranks=2, eps=1e-10, max_iter=3, kind=["exact", "wavy", "exact", "wavy"]),
    "ragged": dict(seed=5, Is=[3, 10, 2, 8], ranks=3, eps=0.0, max_iter=2, kind=["wavy"] * 3),
    "two_modes": dict(seed=12, Is=[12, 9], ranks=4, eps=0.0, max_iter=2, kind=["wavy"] * 3),
    "matrix_arg": dict(seed=2, Is=[7, 8, 9], ranks=3, eps=0.0, max_iter=2, kind=["wavy"] * 2, matrix=True),
    "rank64": dict(seed=3, Is=[64, 64, 4096], ranks=64, eps=0.0, max_iter=1, kind=["rough"] * 2),
}


@pytest.mark.parametrize("name", list(BATCH_CASES))
def test_cross_batch_step_by_step(name, monkeypatch):
    import tntorch_b200 as tnb

    spec = BATCH_CASES[name]
    Is, B, seed = spec["Is"], len(spec["kind"]), spec["seed"]
    axes = _random_axes(Is, seed)
    fn_t, fn_n = _batch_family(torch, spec["kind"]), _batch_family(np, spec["kind"])
    if spec.get("matrix"):
        fns = [(lambda g: (lambda X: g(*X.T)))(fn_t(b)) for b in range(B)]
        probs = [cm.Problem((lambda g: (lambda X: g(*X.T)))(fn_n(b)), domain=axes, function_arg="matrix") for b in range(B)]
    else:
        fns = [fn_t(b) for b in range(B)]
        probs = [cm.Problem(fn_n(b), domain=axes) for b in range(B)]
    rec = Recorder(monkeypatch)
    np.random.seed(seed)
    torch.manual_seed(seed)
    kw = dict(ranks_tt=spec["ranks"], eps=spec["eps"], max_iter=spec["max_iter"])
    t, info = tnb.cross_batch(fns, [torch.as_tensor(a) for a in axes], return_info=True,
                              function_arg="matrix" if spec.get("matrix") else "vectors", **kw)
    steps, picks = rec.of("qr"), rec.of("maxvol")
    np.random.seed(seed)
    torch.manual_seed(seed)
    # the RNG draws of problem b come after those of problems 0..b-1 (cross_batch draws them all up front), so the
    # oracle runs are made in order, each restarted step by step from the device's index sets of its own problem
    dq = dcore = 0.0
    for b in range(B):
        pos = {"s": 0}

        def on_step(kind, j, s, sets):
            nonlocal dq, dcore
            if kind == "F":
                return None
            Qd = steps[pos["s"]][2][b].numpy()
            local_d, Cd = picks[pos["s"]][2][0][b].numpy(), picks[pos["s"]][2][1][b].numpy()
            pos["s"] += 1
            dq = max(dq, np.abs(Qd - s.Q).max())
            assert s.margin > MARGIN and s.cond > COND, (b, kind, j, s.margin, s.cond)
            assert list(local_d) == list(s.local)
            core_d = Cd.reshape(s.core.shape) if kind == "L" else Cd.T.reshape(s.core.shape)
            dcore = max(dcore, _rel(core_d, s.core))
            if kind == "L":
                lr, li = np.divmod(local_d.astype(np.int64), Is[j])
                return np.c_[sets[0][j][lr], li]
            li, lr = np.divmod(local_d.astype(np.int64), s.core.shape[2])
            return np.c_[li, sets[1][j][lr]]

        cores, oi = cm.run(probs[b], ranks_tt=spec["ranks"], eps=spec["eps"], max_iter=spec["max_iter"], on_step=on_step)
        # a frozen problem's cores, index sets and sample count are those of its last active sweep
        assert int(info["iterations"][b]) == len(oi["val_epss"]) and int(info["nsamples"][b]) == oi["nsamples"]
        for n in range(len(Is)):
            assert _note("step_core", _rel(t.cores[n][b].cpu().numpy(), cores[n])) <= TOL["step_core"]
        for n in range(1, len(Is)):
            assert np.array_equal(info["lsets"][n][b].cpu().numpy(), oi["lsets"][n][:, 1:])
        for n in range(len(Is) - 1):
            assert np.array_equal(info["rsets"][n][b].cpu().numpy(), oi["rsets"][n][:, :-1])
    assert _note("step_q", dq) <= TOL["step_q"] and _note("step_core", dcore) <= TOL["step_core"]
    if name == "converge_mixed":
        assert sorted(set(info["iterations"].tolist())) == [1, 3]


def test_cross_batch_refuses_rank_above_64():
    import tntorch_b200 as tnb

    axes = [torch.linspace(0, 1, 70, dtype=torch.float64)] * 3
    with pytest.raises(NotImplementedError):
        tnb.cross_batch([_wavy(torch)], axes, ranks_tt=65, max_iter=1, eps=0.0)


# ================================================================================================ scale through the path
@pytest.mark.parametrize("c", [1e-165, 1e155], ids=["1e-165", "1e155"])
def test_cross_scaled_function(c):
    """cross(c f) = cross(f) with core 0 scaled by c: the QR, maxvol and interpolation cores are scale free."""
    import tntorch_b200 as tnb

    spec = CROSS_DRIVER_CASES["fixed_ranks"]  # every step well conditioned, every decision margin > MARGIN
    axes = [torch.as_tensor(a) for a in _random_axes(spec["Is"], spec["seed"])]
    f = _wavy(torch)
    runs = []
    for s in (1.0, c):
        np.random.seed(spec["seed"])
        torch.manual_seed(spec["seed"])
        runs.append(tnb.cross(lambda *x: s * f(*x), domain=axes, verbose=False, return_info=True, suppress_warnings=True,
                              **spec["kw"]))
    (t0, i0), (t1, i1) = runs
    for a, b in zip(i0["lsets"] + i0["rsets"], i1["lsets"] + i1["rsets"]):
        assert np.array_equal(a, b)
    assert _note("scale_core", _rel(t1.cores[0].cpu().numpy() / c, t0.cores[0].cpu().numpy())) <= TOL["scale_core"]
    for n in range(1, 4):
        assert _note("scale_core", _rel(t1.cores[n].cpu().numpy(), t0.cores[n].cpu().numpy())) <= TOL["scale_core"]
    # The unscaled validation norm of c f under- or overflows, so val_eps is NaN for the scaled problems.  Like
    # cross() (`if val_eps < eps`), cross_batch keeps sweeping on NaN: every problem runs all max_iter sweeps and
    # equals the sequential cross() call of its scaled function.
    bspec = BATCH_CASES["ragged"]
    axes = [torch.as_tensor(a) for a in _random_axes(bspec["Is"], bspec["seed"])]
    fams = [_batch_family(torch, bspec["kind"])(b) for b in range(len(bspec["kind"]))]
    kw = dict(ranks_tt=bspec["ranks"], max_iter=bspec["max_iter"], eps=0.0)
    outs = []
    for s in (1.0, c):
        np.random.seed(bspec["seed"])
        torch.manual_seed(bspec["seed"])
        outs.append(tnb.cross_batch([(lambda g: (lambda *x: s * g(*x)))(g) for g in fams], axes, return_info=True, **kw))
    (b0, j0), (b1, j1) = outs
    assert torch.isnan(j1["val_eps"]).all()
    assert j0["iterations"].tolist() == j1["iterations"].tolist() == [bspec["max_iter"]] * len(fams)
    assert torch.equal(j0["nsamples"], j1["nsamples"])
    np.random.seed(bspec["seed"])
    torch.manual_seed(bspec["seed"])
    for b, g in enumerate(fams):
        t, inf = tnb.cross(lambda *x: c * g(*x), domain=axes, verbose=False, return_info=True, suppress_warnings=True, **kw)
        assert len(inf["val_epss"]) == int(j1["iterations"][b]) and int(inf["nsamples"]) == int(j1["nsamples"][b])
        for n in range(1, len(bspec["Is"])):
            assert np.array_equal(inf["lsets"][n][:, 1:], j1["lsets"][n][b].cpu().numpy())
        for n in range(len(bspec["Is"]) - 1):
            assert np.array_equal(inf["rsets"][n][:, :-1], j1["rsets"][n][b].cpu().numpy())
    for a, b in zip(j0["lsets"][1:] + j0["rsets"][:-1], j1["lsets"][1:] + j1["rsets"][:-1]):
        assert torch.equal(a, b)
    assert _note("scale_core", _rel(b1.cores[0].cpu().numpy() / c, b0.cores[0].cpu().numpy())) <= TOL["scale_core"]
    for n in range(1, len(bspec["Is"])):
        assert _note("scale_core", _rel(b1.cores[n].cpu().numpy(), b0.cores[n].cpu().numpy())) <= TOL["scale_core"]


# ================================================================================================ C ABI
def test_cabi_refusals_leave_outputs_untouched():
    from tntorch_b200._lib import ERR_INVALID, lib

    L = lib()
    A = torch.randn(20, 4, dtype=torch.float64, device="cuda")
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    Q = torch.full((20, 4), 3.5, dtype=torch.float64, device="cuda")
    R = torch.full((4, 4), 3.5, dtype=torch.float64, device="cuda")
    idx = torch.full((32,), -5, dtype=torch.int32, device="cuda")
    Cm = torch.full((20, 32), 3.5, dtype=torch.float64, device="cuda")
    K = torch.full((1,), -5, dtype=torch.int32, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(None)  # noqa: E731
    nb = ws.numel()
    rcs = [
        L.tnb_qr_householder(None, 1, 20, 4, p(ws), nb, p(Q), p(R), None),
        L.tnb_qr_householder(p(A), 1, 20, 4, p(ws), nb, None, p(R), None),
        L.tnb_qr_householder(p(A), 0, 20, 4, p(ws), nb, p(Q), p(R), None),
        L.tnb_qr_householder(p(A), 1, 0, 4, p(ws), nb, p(Q), p(R), None),
        L.tnb_maxvol(None, 1, 20, 4, 1.05, 10, p(ws), nb, p(idx), p(Cm), None, None),
        L.tnb_maxvol(p(A), 1, 20, 4, 1.05, 10, p(ws), nb, None, p(Cm), None, None),
        L.tnb_maxvol(p(A), 1, 0, 4, 1.05, 10, p(ws), nb, p(idx), p(Cm), None, None),
        L.tnb_maxvol(p(A), 1, 20, 0, 1.05, 10, p(ws), nb, p(idx), p(Cm), None, None),
        L.tnb_rect_maxvol(p(A), 1, 20, 4, 1.0, 4, 8, 10, p(ws), nb, p(idx), p(Cm), None, None),
        L.tnb_rect_maxvol(p(A), 1, 4, 4, 1.0, 4, 4, 10, p(ws), nb, p(idx), p(Cm), p(K), None),  # N <= r
        L.tnb_rect_maxvol(p(A), 1, 20, 4, 1.0, 9, 8, 10, p(ws), nb, p(idx), p(Cm), p(K), None),  # minK > maxK
        L.tnb_rect_maxvol(p(A), 1, 20, 4, 1.0, 4, 21, 10, p(ws), nb, p(idx), p(Cm), p(K), None),  # maxK > N
        L.tnb_rect_maxvol(p(A), 1, 20, 4, 1.0, 3, 8, 10, p(ws), nb, p(idx), p(Cm), p(K), None),  # minK < r
        L.tnb_cross_gather_coords(None, None, None, 4, 1, 3, 1, 1, 4, 1, p(Cm), None),
        L.tnb_cross_gather_coords(p(idx), p(idx), p(A), 4, 1, 3, 3, 1, 4, 1, p(Cm), None),  # j >= N
        L.tnb_cross_gather_coords(None, p(idx), p(A), 4, 1, 3, 1, 1, 4, 1, p(Cm), None),  # j > 0 without lsets
        L.tnb_cross_gather_coords(p(idx), p(idx), p(A), 4, 0, 3, 1, 1, 4, 1, p(Cm), None),  # B = 0
        L.tnb_cross_update_lsets(p(idx), None, 1, 1, 1, 4, 2, None, p(K), None),
        L.tnb_cross_update_lsets(p(idx), p(idx), 1, -1, 1, 4, 2, None, p(K), None),
        L.tnb_cross_update_lsets(None, p(idx), 1, 1, 1, 4, 2, None, p(K), None),
        L.tnb_cross_update_rsets(p(idx), p(idx), 1, 3, 0, 4, 1, 2, None, p(K), None),  # j = 0
        L.tnb_cross_update_rsets(p(idx), p(idx), 1, 3, 3, 4, 1, 2, None, p(K), None),  # j >= N
        L.tnb_cross_update_rsets(p(idx), p(idx), 1, 3, 1, 4, 1, 2, None, None, None),
    ]
    ptrs = (C.c_void_p * 2)(A.data_ptr(), A.data_ptr())
    from tntorch_b200._lib import i32

    rcs += [
        L.tnb_cross_tt_eval(None, 2, i32([1, 2, 1]), i32([4, 4]), p(idx), 1, 2, 0, p(Cm), None),
        L.tnb_cross_tt_eval(ptrs, 0, i32([1, 2, 1]), i32([4, 4]), p(idx), 1, 2, 0, p(Cm), None),
        L.tnb_cross_tt_eval(ptrs, 2, i32([1, 2, 1]), i32([4, 4]), None, 1, 2, 0, p(Cm), None),
        L.tnb_cross_tt_eval(ptrs, 2, i32([2, 2, 1]), i32([4, 4]), p(idx), 1, 2, 0, p(Cm), None),
        L.tnb_cross_tt_eval(ptrs, 2, i32([1, 2, 1]), i32([4, 4]), p(idx), 0, 2, 0, p(Cm), None),
    ]
    torch.cuda.synchronize()
    assert rcs == [ERR_INVALID] * len(rcs), rcs
    assert (Q == 3.5).all() and (R == 3.5).all() and (Cm == 3.5).all() and (idx == -5).all() and (K == -5).all()


def test_print_measured():
    """Run last with -s: the largest deviation met per bound across this file (only the tests that ran)."""
    for k in sorted(MEASURED):
        print(f"measured {k}: {MEASURED[k]:.2e} (bound {TOL[k]:.0e})")
