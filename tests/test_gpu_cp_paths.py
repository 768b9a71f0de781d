"""CP-ALS path by path against an fp64 oracle, one sweep at a time.

csrc/cp_als.cuh picks its kernels from the dtype, the shape, the rank and the pointer alignment: the projection of X
(mode N-1 contracted) and of its transposed copy XT (mode N-2 contracted) on the 3xTF32 tensor cores, the FFMA
streaming kernel or the generic GEMM; one of three Khatri-Rao reduction kernels for every further mode contracted; one
of the Jacobi eigensolvers for the normal equations; and, for the HOSVD start, one of three mode-Gram forms with a
Jacobi or a subspace-iteration (ChFSI) eigensolver.  This file
  * restates every one of those choices in Python (the functions under "dispatch", each citing the C++ condition), and
    checks on the CPU that the cases below cover each choice on an SXM (132 SMs) and a PCIe (114 SMs) H100;
  * runs every case from a given start and compares each factor after one sweep, and the error trace of three
    sweeps, with `als_oracle` -- a direct fp64 statement of the ALS sweep that shares no code with the kernels or with
    tests/cp_tree_model.py;
  * checks the HOSVD start against np.linalg.eigh, the singular and zero edges, the C ABI's buffer bounds, and two
    host threads on two streams.
Factor deviations are bounded by c * max(1, kappa), kappa the largest condition number of the normal-equation matrices
P_n the oracle meets (each case asserts kappa <= 30, so the bound cannot turn vacuous).  Run with -s to see the
measured deviations."""
import ctypes as C
import threading

import numpy as np
import pytest
import torch

EPS64 = 2.220446049250313e-16
NP_DTYPE = {torch.float64: np.float64, torch.float32: np.float32}
DTYPES = [torch.float64, torch.float32]
IDS = ["f64", "f32"]
KAPPA_MAX = 30.0
# factor: (a), factor deviation <= c * max(1, kappa) after one sweep; sweeps3: the same after the HOSVD start and
# three sweeps; trace: (b), |error trace - oracle| and |errors[-1] - true reconstruction error|; subspace / chfsi: the
# HOSVD start against eigh with the Jacobi / the ChFSI eigensolver.  Each bound is at most 10x the largest deviation
# measured on an H100 SXM (132 SMs, 700 W) over the cases here, printed with -s:
#   fp64: factor 7.2e-14 (wrap_f64), sweeps3 1.3e-12, trace 1.3e-14, subspace 5.4e-14, chfsi 8.2e-14;
#   fp32: factor 6.0e-7 (n2_tc_f32: the 3xTF32 projection, then a 20000-term fp32 GEMM), sweeps3 2.6e-8, trace 5.7e-6
#         (tc_both_xoff_f32: the Gram-form error of fp32 factors), subspace 6.1e-8, chfsi 2.2e-6.
TOL = {
    torch.float64: dict(factor=5e-13, sweeps3=1e-11, trace=1e-13, subspace=5e-13, chfsi=5e-13),
    torch.float32: dict(factor=3e-6, sweeps3=2e-7, trace=1e-5, subspace=5e-7, chfsi=2e-5),
}


# ==================================================================================================== fp64 oracle
def _operands(A, skip):
    ops = []
    for m, a in enumerate(A):
        if m != skip:
            ops += [a, [m, len(A)]]
    return ops


def mttkrp(X, A, n):
    """M_n = X_(n) (Khatri-Rao product of the factors other than n), as one einsum in integer-sublist form (any N)."""
    N = X.ndim
    return np.einsum(X, list(range(N)), *_operands(A, n), [n, N], optimize=True)


def reconstruct(A):
    N = len(A)
    return np.einsum(*_operands(A, -1), list(range(N)), optimize=True)


def _kappa(P, rcond):
    """lambda_max / smallest eigenvalue the pseudo-inverse keeps (1 for P = 0)."""
    w = np.linalg.eigvalsh(P)
    if w[-1] <= 0:
        return 1.0
    kept = w[w > rcond * w[-1]]
    return float(w[-1] / kept.min())


def als_oracle(X, A0, sweeps):
    """`sweeps` Gauss-Seidel ALS sweeps from A0 in fp64: A_n = M_n pinv(P_n, rcond = R eps), P_n the Hadamard product of
    the other A_m^T A_m.  Returns the factors after each sweep, the Gram-form error after each sweep, kappa(P_n) of
    every update, and the true reconstruction error of the final factors."""
    X = np.asarray(X, dtype=np.float64)
    N, R = X.ndim, A0[0].shape[1]
    A = [np.array(a, dtype=np.float64) for a in A0]
    G = [a.T @ a for a in A]
    rcond = R * EPS64
    normX2 = float(np.vdot(X, X))
    out = dict(factors=[], errors=[], kappa=[])
    for _ in range(sweeps):
        for n in range(N):
            M = mttkrp(X, A, n)
            P = np.ones((R, R))
            for m in range(N):
                if m != n:
                    P = P * G[m]
            out["kappa"].append(_kappa(P, rcond))
            A[n] = M @ np.linalg.pinv(P, rcond=rcond, hermitian=True)
            G[n] = A[n].T @ A[n]
        Pall = np.ones((R, R))
        for g in G:
            Pall = Pall * g
        e2 = max(normX2 - 2.0 * float(np.sum(M * A[N - 1])) + float(Pall.sum()), 0.0)
        out["errors"].append(np.sqrt(e2 / normX2) if normX2 > 0 else 0.0)
        out["factors"].append([a.copy() for a in A])
    out["recon"] = _relerr(X, A)
    return out


def _relerr(X, A):
    nx = np.linalg.norm(X)
    return float(np.linalg.norm(X - reconstruct(A)) / nx) if nx > 0 else 0.0


# ==================================================================================================== dispatch
# Each function restates one choice of the device code for a case; `sms` is the usable SM count
# (cudaDevAttrMultiProcessorCount minus tnb_set_reserved_sms, common.cuh:153-159).
PROJ_TC_MIN_ROWS = 16384  # sweep.cuh:37
PT_MAX_N = 64  # project_tc.cuh:46
JACOBI_MAX_N = 256  # jacobi.cuh:9
REDUCE_CAP = 8192 * 256  # khatri_reduce_kernel: grid_for(L*Q*R, 256, 8192), cp_als.cuh:307
REDUCE2_CAP = 16384 * 256  # khatri_reduce2_kernel: grid_for(L*Q*R/2, 256, 16384), cp_als.cuh:303


def tc_workspace(dtype, shape, R):
    """cp_als.cuh:394-397: the tensor-core projection gets a workspace when an fp32 projection's K (I_{N-1}, and for
    N >= 3 also I_{N-2}) has K % 4 == 0, K >= 32 and R <= 64."""
    N = len(shape)
    return dtype == torch.float32 and any(R <= PT_MAX_N and shape[m] % 4 == 0 and shape[m] >= 32
                                          for m in range(N - 2 if N >= 3 else N - 1, N))


def project_kernel(dtype, rows, K, R, a_aligned16, tc_ws):
    """project_any, sweep.cuh:43-53 (C is the workspace, always 256-byte aligned):
    tc:      tc_ws && rows >= 16384 && project_tc_shape_ok (R <= 64, K % 4 == 0, 32 <= K <= 2^24, 128 <= rows < 2^31-256,
             A 16-byte aligned; project_tc.cuh:390-395);
    ffma:    fp32 && project_f32_fast_ok (1 <= R <= 64, K % 4 == 0, 4 <= K < 2^31, A 16-byte aligned; project.cuh:120-123);
    generic: gemm_direct otherwise."""
    f32 = dtype == torch.float32
    if (f32 and tc_ws and rows >= PROJ_TC_MIN_ROWS and R <= PT_MAX_N and K % 4 == 0 and 32 <= K <= 1 << 24
            and 128 <= rows < (1 << 31) - 256 and a_aligned16):
        return "tc"
    if f32 and 1 <= R <= 64 and K % 4 == 0 and 4 <= K < 1 << 31 and a_aligned16:
        return "ffma"
    return "generic"


def projections(case):
    """{"X": (kernel, rows, K), "XT": ...}.  N >= 3 (cp_tree_mttkrp): X projects mode N-1 for mode 0 (cp_als.cuh:315),
    XT (workspace, [I_{N-1}, I_0..I_{N-2}]) projects mode N-2 for mode N-1 (cp_als.cuh:342).  N == 2 (cp_mttkrp): X
    projects mode 1 for mode 0 (cp_als.cuh:221); mode 1 is a first-mode gemm_direct (cp_als.cuh:227), not a projection."""
    shape, R, dtype = case["shape"], case["R"], case["dtype"]
    N, numel = len(shape), int(np.prod(shape))
    ws = tc_workspace(dtype, shape, R)
    x16 = case.get("xoff", 0) * np.dtype(NP_DTYPE[dtype]).itemsize % 16 == 0
    out = {"X": (project_kernel(dtype, numel // shape[-1], shape[-1], R, x16, ws), numel // shape[-1], shape[-1])}
    if N >= 3:
        out["XT"] = (project_kernel(dtype, numel // shape[-2], shape[-2], R, True, ws), numel // shape[-2], shape[-2])
    return out


def khatri_kernel(dtype, L, I, Q, R, al8, sms):
    """cp_khatri, cp_als.cuh:294-308: fp32 with an even R and Y, A, out 8-byte aligned -> the split kernel when
    L*Q*R/2 < sms*256, else khatri_reduce2_kernel; everything else khatri_reduce_kernel."""
    if dtype == torch.float32 and R % 2 == 0 and al8:
        return "split" if L * Q * (R // 2) < sms * 256 else "reduce2"
    return "reduce"


def reductions(case, sms):
    """Every cp_khatri call of one sweep, as dicts (mode, kernel, L, I, Q, wrap) (cp_tree_mttkrp, cp_als.cuh:310-352).
    Y, out and the chain buffers are workspace (256-byte aligned); A is a factor, at factor_offset bytes past the
    buffer's alignment (the factor offsets are multiples of 64 elements, cp_als.cuh:204).  N == 2 has none."""
    shape, R, dtype = case["shape"], case["R"], case["dtype"]
    N = len(shape)
    al8 = case.get("foff", 0) % 8 == 0
    left = [int(np.prod(shape[:k])) for k in range(N)]
    calls = []

    def add(n, L, I, Q):
        k = khatri_kernel(dtype, L, I, Q, R, al8, sms)
        wrap = (k == "reduce" and L * Q * R > REDUCE_CAP) or (k == "reduce2" and L * Q * (R // 2) > REDUCE2_CAP)
        calls.append(dict(mode=n, kernel=k, L=L, I=I, Q=Q, wrap=wrap))

    if N < 3:
        return calls
    for k in range(N - 3, -1, -1):  # mode 0: the right-to-left chain, cp_als.cuh:317-321
        add(0, left[k + 1], shape[k + 1], 1)
    for n in range(1, N - 1):  # modes 1..N-2: reduce modes 0..n-1 of chain[n] (or Y), cp_als.cuh:328-339
        for lo in range(n):
            add(n, 1, shape[lo], int(np.prod(shape[lo + 1: n + 1])))
    for m in range(N - 3, -1, -1):  # mode N-1: XT's projection reduced over modes N-3..0, cp_als.cuh:344-350
        add(N - 1, shape[N - 1] * left[m], shape[m], 1)
    return calls


def solver(R):
    """The eigen-solve of P (R x R fp64) behind A_n = M P^+ (cp_als.cuh:519):
    jacobi2_eigh (jacobi2.cuh:363-389): 8 <= R <= 64 the mixed fp32/fp64 kernel, other R <= 80 the fp64 kernel;
    above 80 jacobi_eigh (jacobi.cuh:301-308): A and V in shared memory while 2*np*(np+8) doubles fit in
    2*104*112 (R <= 104), A alone while np*(np+8) does (R <= 148), global memory up to 256; R > 256 is refused."""
    np_ = R + (R & 1)
    if R < 1 or R > JACOBI_MAX_N:
        return None
    if R <= 80:
        return "jacobi2_mixed" if 8 <= R <= 64 else ("jacobi2_f64_small" if R < 8 else "jacobi2_f64_wide")
    maxb = 2 * 104 * 112
    if 2 * np_ * (np_ + 8) <= maxb:
        return "jacobi_smem_AV"
    if np_ * (np_ + 8) <= maxb:
        return "jacobi_smem_A"
    return "jacobi_global"


def start_forms(shape, R):
    """HOSVD start per mode (cp_als.cuh:444-487): the mode Gram as C^T C of X viewed (rest x I) for the last mode,
    C C^T of X viewed (I x rest) when left[n] == 1, else a batched sum over the left index; Jacobi (all eigenpairs) for
    I <= 256, else ChFSI for the min(R, I) leading ones (eig_carve, sweep.cuh:195-223); pseudo-random columns past
    min(R, I) (cp_init_factor_kernel)."""
    N = len(shape)
    out = []
    for n, I in enumerate(shape):
        form = "last" if n == N - 1 else ("left1" if int(np.prod(shape[:n])) == 1 else "batched")
        out.append(dict(form=form, eig="jacobi" if I <= JACOBI_MAX_N else "chfsi", random=max(R - I, 0)))
    return out


# ==================================================================================================== cases
def _case(shape, R, dtype, **kw):
    return dict(shape=tuple(shape), R=R, dtype=dtype, **kw)


F32, F64 = torch.float32, torch.float64
N16 = (2, 3, 2, 2, 3, 2, 2, 2, 3, 2, 2, 2, 3, 2, 2, 2)  # 2^12 * 3^4 = 331776 elements
# name -> case.  start: "gauss" (true factors and start Gaussian) or "ortho" (orthonormal columns where I_n >= R, unit-norm
# columns elsewhere); xoff: X passed at this many elements past a 256-byte boundary.
CASES = {
    "n2_f64": _case((30, 20), 3, F64),
    "n2_f32": _case((30, 20), 3, F32),
    "n2_tc_f32": _case((20000, 36), 8, F32),
    "ffma_split_f32": _case((20, 12, 16), 8, F32),
    "small_f64": _case((20, 18, 16), 8, F64),
    "odd_r_f32": _case((21, 19, 13), 5, F32),
    "odd_r_f64": _case((21, 19, 13), 5, F64),
    "r64_f32": _case((40, 36, 27, 44), 64, F32),
    "tc_both_f32": _case((20, 26, 40, 36), 16, F32),
    "tc_both_xoff_f32": _case((20, 26, 40, 36), 16, F32, xoff=1),
    "wrap_f64": _case((200, 200, 8, 8), 64, F64, start="ortho"),
    "wrap_f32": _case((400, 352, 8, 8), 64, F32, start="ortho"),
    "r72_f64": _case((80, 76, 6), 72, F64, start="ortho"),
    "r72_f32": _case((80, 76, 6), 72, F32, start="ortho"),
    "r96_f64": _case((100, 98, 5), 96, F64, start="ortho"),
    "r96_f32": _case((100, 98, 5), 96, F32, start="ortho"),
    "r130_f64": _case((140, 136, 4), 130, F64, start="ortho"),
    "r130_f32": _case((140, 136, 4), 130, F32, start="ortho"),
    # a mode above 256 would be refused at R = 256: the workspace query sizes the HOSVD start's ChFSI scratch (target
    # rank <= 240) even when a start is given
    "r256_f64": _case((256, 256, 4), 256, F64, start="ortho"),
    "r256_f32": _case((256, 256, 4), 256, F32, start="ortho"),
    "n5_f64": _case((8, 7, 6, 5, 9), 4, F64, start="ortho"),
    "n5_f32": _case((8, 7, 6, 5, 9), 4, F32, start="ortho"),
    "unit_front_mid_f64": _case((1, 7, 1, 9, 5), 3, F64),
    "unit_front_mid_f32": _case((1, 7, 1, 9, 5), 3, F32),
    "unit_end_f64": _case((6, 5, 1), 2, F64),
    "unit_end_f32": _case((6, 5, 1), 2, F32),
    "n16_f64": _case(N16, 2, F64, start="ortho"),
    "n16_f32": _case(N16, 2, F32, start="ortho"),
}
# the factors at a 4-byte offset (C ABI only, test_misaligned_factors_match_oracle): cp_khatri takes the scalar kernel
MISALIGNED_FACTORS = _case((24, 20, 18), 8, F32, foff=4)


def _sweep_cases():
    return list(CASES.values()) + [MISALIGNED_FACTORS]


def _coverage(sms):
    seen = set()
    for c in _sweep_cases():
        for side, (k, _, _) in projections(c).items():
            seen.add(("proj", side, k))
        for call in reductions(c, sms):
            seen.add(("reduce", call["kernel"]))
            if call["I"] >= 8 and call["I"] % 8:
                seen.add(("reduce_tail", call["kernel"]))
            if call["wrap"]:
                seen.add(("wrap", call["kernel"]))
        seen.add(("solver", solver(c["R"])))
        seen.add(("N", len(c["shape"])))
        sh = c["shape"]
        if sh[0] == 1:
            seen.add(("unit", "front"))
        if any(s == 1 for s in sh[1:-1]):
            seen.add(("unit", "middle"))
        if sh[-1] == 1:
            seen.add(("unit", "end"))
        if any(c["R"] > s for s in sh):
            seen.add(("R>I",))
    return seen


@pytest.mark.parametrize("sms", [132, 114])
def test_cases_cover_every_dispatch_choice(sms):
    """CPU: the case list reaches every projection kernel on each side, every reduction kernel (each with a row count
    past the 8-row unroll that leaves a tail), both grid-stride wraps, every solver range, N = 2..5 and 16, size-1
    modes at either end and in the middle, and R > I_n -- on an SXM and a PCIe H100 (the split threshold moves)."""
    seen = _coverage(sms)
    want = {("proj", side, k) for side in ("X", "XT") for k in ("tc", "ffma", "generic")}
    want |= {("reduce", k) for k in ("split", "reduce2", "reduce")} | {("reduce_tail", k) for k in ("split", "reduce2", "reduce")}
    want |= {("wrap", "reduce"), ("wrap", "reduce2")}
    want |= {("solver", s) for s in ("jacobi2_f64_small", "jacobi2_mixed", "jacobi2_f64_wide", "jacobi_smem_AV",
                                     "jacobi_smem_A", "jacobi_global")}
    want |= {("N", n) for n in (2, 3, 4, 5, 16)} | {("unit", w) for w in ("front", "middle", "end")} | {("R>I",)}
    assert not want - seen, sorted(want - seen)


def test_dispatch_restatement_spot_checks():
    """CPU: the restatement gives what the case comments claim, at both SM counts."""
    for sms in (132, 114):
        p = projections(CASES["r64_f32"])
        assert p["X"][0] == "tc" and p["XT"][0] == "generic"
        assert projections(CASES["tc_both_f32"])["XT"][0] == "tc" and projections(CASES["tc_both_f32"])["X"][0] == "tc"
        p = projections(CASES["tc_both_xoff_f32"])
        assert p["X"][0] == "generic" and p["XT"][0] == "tc"  # a 4-byte aligned X declines TC and FFMA
        assert projections(CASES["n2_tc_f32"])["X"][0] == "tc"
        assert {c["kernel"] for c in reductions(MISALIGNED_FACTORS, sms)} == {"reduce"}
        assert {c["kernel"] for c in reductions(CASES["odd_r_f32"], sms)} == {"reduce"}
        assert [c for c in reductions(CASES["wrap_f64"], sms) if c["wrap"]]
        assert [c for c in reductions(CASES["wrap_f32"], sms) if c["wrap"] and c["kernel"] == "reduce2"]
        assert start_forms((300, 24, 20), 6)[0]["eig"] == "chfsi"
        assert start_forms((1, 30, 20, 16), 4)[1]["form"] == "left1"
    # (40, 36, 27, 44) R = 64, mode 2: L*Q*R/2 = 31104 pairs, split on 132 SMs (33792), not on 114 (29184)
    k132 = [c["kernel"] for c in reductions(CASES["r64_f32"], 132) if c["mode"] == 2 and c["I"] == 40]
    k114 = [c["kernel"] for c in reductions(CASES["r64_f32"], 114) if c["mode"] == 2 and c["I"] == 40]
    assert k132 == ["split"] and k114 == ["reduce2"]
    assert solver(257) is None


# ==================================================================================================== inputs
def _cond_factor(G, ortho):
    if not ortho:
        return G
    if G.shape[0] >= G.shape[1]:
        return np.linalg.qr(G)[0]
    return G / np.linalg.norm(G, axis=0)


def _problem(case, seed):
    """(X, A0) in fp64: X a rank-R CP tensor plus 10 % noise, A0 its factors plus 30 % noise.  Size-1 modes carry
    entries near 1 (a 1 x R factor's Gram is rank 1: P_n = diag(a) B diag(a) stays as well conditioned as B)."""
    rng = np.random.default_rng(seed)
    ortho = case.get("start") == "ortho"
    F, A0 = [], []
    for I in case["shape"]:
        if I == 1:
            f = 1.0 + 0.2 * rng.standard_normal((1, case["R"]))
            a = f + 0.1 * rng.standard_normal(f.shape)
        else:
            f = _cond_factor(rng.standard_normal((I, case["R"])), ortho)
            a = _cond_factor(f + 0.3 * rng.standard_normal(f.shape) / (np.sqrt(I) if ortho else 1.0), ortho)
        F.append(f)
        A0.append(a)
    X = reconstruct(F)
    X = X + 0.1 * np.linalg.norm(X) / np.sqrt(X.size) * rng.standard_normal(X.shape)
    return X, A0


def _on_device(case, X, A0):
    """(X on the device in the case's dtype, maybe at an element offset; A0 on the device; both as fp64 NumPy values)."""
    dt = case["dtype"]
    Xc = np.ascontiguousarray(X, dtype=NP_DTYPE[dt])
    A0c = [np.ascontiguousarray(a, dtype=NP_DTYPE[dt]) for a in A0]
    off = case.get("xoff", 0)
    if off:
        buf = torch.zeros(Xc.size + off, dtype=dt, device="cuda")
        buf[off:] = torch.as_tensor(Xc.reshape(-1))
        Xd = buf[off:].view(Xc.shape)
        assert Xd.is_contiguous() and Xd.data_ptr() % 16 == off * Xc.itemsize % 16
    else:
        Xd = torch.as_tensor(Xc).cuda()
    return Xd, [torch.as_tensor(a).cuda() for a in A0c], Xc.astype(np.float64), [a.astype(np.float64) for a in A0c]


def _host(factors):
    return [f.detach().cpu().numpy().astype(np.float64) for f in factors]


def _factor_dev(lib, ref):
    return max(float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)) for a, b in zip(lib, ref))


def _sms():
    from tntorch_b200 import ops

    ops.set_reserved_sms(0)
    return torch.cuda.get_device_properties(0).multi_processor_count


def _seed(name):
    return sum(ord(c) * (i + 1) for i, c in enumerate(name)) % 10007


# ==================================================================================================== sweeps
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_sweep_matches_oracle(name):
    """(a) every factor after one sweep; (b) the error trace of three sweeps and its last value against the true
    reconstruction error; (c) X and A0 unchanged; (d) two identical calls are bitwise equal."""
    from tntorch_b200 import ops

    case = CASES[name]
    sms = _sms()
    dt, R = case["dtype"], case["R"]
    tol = TOL[dt]
    X, A0 = _problem(case, _seed(name))
    Xd, A0d, X64, A064 = _on_device(case, X, A0)
    Xbefore, Abefore = Xd.clone(), [a.clone() for a in A0d]
    orc = als_oracle(X64, A064, 3)
    kappa = max(orc["kappa"])
    assert kappa <= KAPPA_MAX, (name, kappa, "the case is not as well conditioned as it is built to be")

    one = ops.cp_als(Xd, R, max_iter=1, tol=float("-inf"), init=A0d)
    three, info = ops.cp_als(Xd, R, max_iter=3, tol=float("-inf"), init=A0d, return_info=True)
    again, info2 = ops.cp_als(Xd, R, max_iter=3, tol=float("-inf"), init=A0d, return_info=True)
    torch.cuda.synchronize()
    dev = _factor_dev(_host(one), orc["factors"][0])
    trace = max(abs(a - b) for a, b in zip(info["errors"], orc["errors"]))
    recon = abs(info["errors"][-1] - _relerr(X64, _host(three)))
    paths = dict(projections(dict(case)), reduce=sorted({c["kernel"] for c in reductions(case, sms)}), solver=solver(R))
    print(f"{name}: sms {sms} {paths}; kappa {kappa:.2f}; factor dev {dev:.2e} (tol {tol['factor'] * kappa:.1e}), "
          f"trace dev {trace:.2e}, errors[-1] vs reconstruction {recon:.2e} (tol {tol['trace']:.0e}); "
          f"errors {info['errors']}, oracle {orc['errors']}")
    assert info["iters"] == 3 and len(info["errors"]) == 3
    assert dev <= tol["factor"] * max(1.0, kappa), (name, dev)  # (a)
    assert trace <= tol["trace"], (name, info["errors"], orc["errors"])  # (b)
    assert recon <= tol["trace"], (name, recon)
    assert torch.equal(Xd, Xbefore) and all(torch.equal(a, b) for a, b in zip(A0d, Abefore)), "input modified"  # (c)
    # (d) the factors are bitwise repeatable; the error trace may differ in its last bits (cp_error_terms_kernel sums
    # its block partials with atomics, and feeds only the error)
    assert all(torch.equal(a, b) for a, b in zip(three, again)), "factors not deterministic"
    assert max(abs(a - b) for a, b in zip(info["errors"], info2["errors"])) <= 5e-14, (info["errors"], info2["errors"])


_KERNELS = {
    "project_tc_kernel": ("proj", "tc"), "project_f32_kernel": ("proj", "ffma"),
    "khatri_reduce2_split_kernel": ("reduce", "split"), "khatri_reduce2_kernel": ("reduce", "reduce2"),
    "khatri_reduce_kernel": ("reduce", "reduce"), "jacobi2_mixed_kernel": ("solver", "jacobi2_mixed"),
    "jacobi2_eigh_kernel<double>": ("solver", "jacobi2_f64"), "jacobi_eigh_kernel<double, true": ("solver", "jacobi_smem"),
    "jacobi_eigh_kernel<double, false": ("solver", "jacobi_global"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in CASES if not n.startswith("n16") and not n.startswith("r256")])
def test_dispatch_restatement_matches_launched_kernels(name):
    """The kernels one sweep launches (torch.profiler) are the ones the restatement names: the projection kernels that
    are not the generic GEMM, the Khatri-Rao reductions, and the eigensolver of the normal equations."""
    from torch.profiler import ProfilerActivity, profile

    from tntorch_b200 import ops

    case = CASES[name]
    sms = _sms()
    X, A0 = _problem(case, _seed(name))
    Xd, A0d, _, _ = _on_device(case, X, A0)
    ops.cp_als(Xd, case["R"], max_iter=1, tol=float("-inf"), init=A0d)  # first-call attribute setup out of the trace
    torch.cuda.synchronize()
    names = []
    for _ in range(3):  # the activity trace occasionally comes back empty: take it again, never accept an empty one
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            ops.cp_als(Xd, case["R"], max_iter=1, tol=float("-inf"), init=A0d)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        if names:
            break
    assert names, "the profiler recorded no kernel"
    seen = {what for n in names for key, what in _KERNELS.items() if key in n}
    s = solver(case["R"])
    want = {("proj", k) for k, _, _ in projections(case).values() if k != "generic"}
    want |= {("reduce", c["kernel"]) for c in reductions(case, sms)}
    want.add(("solver", {"jacobi2_f64_small": "jacobi2_f64", "jacobi2_f64_wide": "jacobi2_f64", "jacobi_smem_AV": "jacobi_smem",
                         "jacobi_smem_A": "jacobi_smem"}.get(s, s)))
    print(f"{name}: sms {sms}, launched {sorted(seen)}")
    assert seen == want, (name, sorted(seen), sorted(want))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_limits_raise(dtype):
    from tntorch_b200 import ops

    X = torch.randn(300, 280, 2, dtype=dtype, device="cuda")
    with pytest.raises(ValueError):  # R above the eigensolver's 256 is refused by the sizing query
        ops.cp_als(X, 257, max_iter=1)
    X17 = torch.randn((2,) * 17, dtype=dtype, device="cuda")
    with pytest.raises(ValueError):
        ops.cp_als(X17, 2, max_iter=1)


# ==================================================================================================== edges
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("R", [6, 12])
def test_singular_normal_equations_give_the_minimum_norm_solution(R, dtype):
    """A0 with column 1 equal to column 0 in every factor: every P_n is singular, the two columns stay equal and the
    factors match the oracle's minimum-norm (pinv) solution.  R = 6 runs the fp64 Jacobi, R = 12 the mixed one."""
    from tntorch_b200 import ops

    case = _case((14, 12, 10), R, dtype)
    X, A0 = _problem(case, 400 + R)
    for a in A0:
        a[:, 1] = a[:, 0]
    Xd, A0d, X64, A064 = _on_device(case, X, A0)
    orc = als_oracle(X64, A064, 1)
    kappa = max(orc["kappa"])  # over the range P keeps
    assert kappa <= KAPPA_MAX, kappa
    out = _host(ops.cp_als(Xd, R, max_iter=1, tol=float("-inf"), init=A0d))
    dev = _factor_dev(out, orc["factors"][0])
    split = max(float(np.linalg.norm(a[:, 0] - a[:, 1]) / np.linalg.norm(a)) for a in out)
    print(f"duplicated column R={R} {dtype}: solver {solver(R)}, kappa {kappa:.2f}, factor dev {dev:.2e}, "
          f"column split {split:.2e}")
    assert all(np.isfinite(a).all() for a in out)
    assert dev <= TOL[dtype]["factor"] * max(1.0, kappa), dev
    assert split <= TOL[dtype]["factor"], split


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_zero_column_stays_zero(dtype):
    """A zero column in the last factor zeroes that column of every P_n's Hadamard product: it stays zero in every
    factor, with no NaN, and the other columns match the oracle."""
    from tntorch_b200 import ops

    R = 6
    case = _case((14, 12, 10), R, dtype)
    X, A0 = _problem(case, 410)
    A0[-1][:, 2] = 0.0
    Xd, A0d, X64, A064 = _on_device(case, X, A0)
    orc = als_oracle(X64, A064, 2)
    out = _host(ops.cp_als(Xd, R, max_iter=2, tol=float("-inf"), init=A0d))
    kappa = max(orc["kappa"])
    dev = _factor_dev(out, orc["factors"][-1])
    col = max(float(np.abs(a[:, 2]).max()) for a in out)
    print(f"zero column {dtype}: kappa {kappa:.2f}, factor dev {dev:.2e}, largest entry of the zero column {col:.1e}")
    assert all(np.isfinite(a).all() for a in out)
    assert col == 0.0
    # NumPy's pinv (Householder tridiagonalisation) leaks ~1e-16 into the zero direction
    assert all(np.abs(a[:, 2]).max() <= 1e-13 * np.abs(a).max() for a in orc["factors"][-1])
    assert dev <= TOL[dtype]["factor"] * max(1.0, kappa), dev


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_zero_tensor(dtype):
    """X = 0 from the default start (Jacobi on zero mode Grams): finite factors and an error of exactly 0 (the library
    returns 0 for ||X|| = 0, cp_als.cuh:540)."""
    from tntorch_b200 import ops

    X = torch.zeros(10, 9, 8, dtype=dtype, device="cuda")
    fac, info = ops.cp_als(X, 3, max_iter=3, tol=float("-inf"), return_info=True)
    assert all(torch.isfinite(f).all() for f in fac)
    assert info["errors"] == [0.0, 0.0, 0.0], info


# ==================================================================================================== HOSVD start
def _signal(shape, R, seed, noise=1e-3):
    """Orthonormal-column factors, column r scaled by 0.75^r (eigenvalue ratios 0.56 between consecutive columns), plus
    `noise` relative Gaussian noise."""
    rng = np.random.default_rng(seed)
    F = []
    for I in shape:
        G = rng.standard_normal((I, R))
        F.append(np.linalg.qr(G)[0] if I >= R else G / np.linalg.norm(G, axis=0))
    F[0] = F[0] * 0.75 ** np.arange(R)
    X = reconstruct(F)
    return X + noise * np.linalg.norm(X) / np.sqrt(X.size) * rng.standard_normal(X.shape)


def _start_dev(X64, fac, R):
    """Per mode: (spectral norm of the projector difference, largest column deviation up to sign over the columns whose
    eigenvalue is >= 10 % away from both neighbours) between the first min(R, I) columns and eigh of X_(n) X_(n)^T."""
    out = []
    for n, A in enumerate(fac):
        I = A.shape[0]
        k = min(R, I)
        Xn = np.moveaxis(X64, n, 0).reshape(I, -1)
        w, V = np.linalg.eigh(Xn @ Xn.T)
        w, V = w[::-1], V[:, ::-1]
        U, E = A[:, :k], V[:, :k]
        sub = float(np.linalg.norm(U @ U.T - E @ E.T, 2))
        col = 0.0
        for j in range(k):
            gaps = [abs(w[j] - w[i]) / max(w[j], w[i]) for i in (j - 1, j + 1) if 0 <= i < I]
            if w[j] > 0 and all(g >= 0.1 for g in gaps):
                col = max(col, min(np.linalg.norm(U[:, j] - E[:, j]), np.linalg.norm(U[:, j] + E[:, j])))
        out.append((sub, col))
    return out


HOSVD = {
    "forms": dict(shape=(24, 20, 18), R=4),  # left1, batched, last
    "leading_unit": dict(shape=(1, 30, 20, 16), R=4),  # mode 1 has left[1] == 1; mode 0 has I < R
    "chfsi": dict(shape=(300, 24, 20), R=6),  # mode 0: I > 256, the subspace-iteration start
}


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("name", list(HOSVD))
def test_hosvd_start_matches_eigh(name, dtype):
    from tntorch_b200 import ops

    spec = HOSVD[name]
    shape, R = spec["shape"], spec["R"]
    X = _signal(shape, R, 500 + len(shape))
    Xc = X.astype(NP_DTYPE[dtype])
    fac = _host(ops.cp_als(torch.as_tensor(Xc).cuda(), R, max_iter=0))
    forms = start_forms(shape, R)
    devs = _start_dev(Xc.astype(np.float64), fac, R)
    for n, ((sub, col), f) in enumerate(zip(devs, forms)):
        t = TOL[dtype]["chfsi" if f["eig"] == "chfsi" else "subspace"]
        print(f"hosvd {name} {dtype} mode {n} ({f['form']}, {f['eig']}): subspace {sub:.2e}, column {col:.2e} (tol {t:.0e})")
    for n, ((sub, col), f) in enumerate(zip(devs, forms)):
        t = TOL[dtype]["chfsi" if f["eig"] == "chfsi" else "subspace"]
        assert sub <= t and col <= t, (name, n, f, sub, col)
        if f["random"]:
            extra = fac[n][:, shape[n]:]
            assert np.all(np.abs(extra) < 1.0), (name, n)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_hosvd_random_columns_are_bounded_and_repeatable(dtype):
    """R > I_n: the columns past I_n are pseudo-random in (-1, 1) and the same on every call."""
    from tntorch_b200 import ops

    X = torch.as_tensor(_signal((4, 9, 8), 6, 520).astype(NP_DTYPE[dtype])).cuda()
    a = ops.cp_als(X, 6, max_iter=0)
    b = ops.cp_als(X, 6, max_iter=0)
    extra = a[0][:, 4:]
    assert torch.equal(extra, b[0][:, 4:]) and bool((extra.abs() < 1).all()) and bool((extra != 0).any())
    assert all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("name", list(HOSVD))
def test_default_start_then_sweeps_match_oracle(name, dtype):
    """cp_als(X, R, max_iter=3) from the default start equals the oracle's three sweeps from that call's own
    max_iter=0 output."""
    from tntorch_b200 import ops

    spec = HOSVD[name]
    X = _signal(spec["shape"], spec["R"], 530 + len(spec["shape"]), noise=0.1)
    Xd = torch.as_tensor(X.astype(NP_DTYPE[dtype])).cuda()
    start = _host(ops.cp_als(Xd, spec["R"], max_iter=0))
    fac, info = ops.cp_als(Xd, spec["R"], max_iter=3, tol=float("-inf"), return_info=True)
    orc = als_oracle(Xd.double().cpu().numpy(), start, 3)
    kappa = max(orc["kappa"])
    dev = _factor_dev(_host(fac), orc["factors"][-1])
    trace = max(abs(a - b) for a, b in zip(info["errors"], orc["errors"]))
    print(f"default start {name} {dtype}: kappa {kappa:.2f}, factor dev after 3 sweeps {dev:.2e}, trace dev {trace:.2e}")
    assert kappa <= KAPPA_MAX, kappa
    assert dev <= TOL[dtype]["sweeps3"] * max(1.0, kappa), dev
    assert trace <= TOL[dtype]["trace"], (info["errors"], orc["errors"])


# ==================================================================================================== C ABI, streams
CANARY = 1 << 20


def _guarded(nbytes):
    """A device byte buffer of exactly `nbytes` followed by a 1 MiB canary; returns (buffer, canary pattern)."""
    pattern = ((torch.arange(CANARY, device="cuda") * 151 + 89) % 256).to(torch.uint8)
    buf = torch.empty(nbytes + CANARY, dtype=torch.uint8, device="cuda")
    buf[nbytes:] = pattern
    return buf, pattern


def _intact(buf, nbytes, pattern):
    torch.cuda.synchronize()
    return torch.equal(buf[nbytes:], pattern)


def _cabi_run(case, X64, A064, max_iter, factor_byte_offset=0):
    """tnb_cp_als (A064 None: the HOSVD start) or tnb_cp_als_from through ctypes, with a workspace of exactly
    tnb_cp_als_workspace_bytes and a factors buffer of exactly the queried capacity (at `factor_byte_offset` past a
    256-byte boundary), each followed by a canary, and NaN in the padding between factors.  Returns the factors as
    fp64 NumPy arrays after checking both canaries and the padding."""
    from tntorch_b200 import _lib

    L = _lib.lib()
    dt = case["dtype"]
    code, esz = (_lib.TNB_F64, 8) if dt == torch.float64 else (_lib.TNB_F32, 4)
    shape, R = case["shape"], case["R"]
    N = len(shape)
    sh = _lib.i64(shape)
    offs = (C.c_int64 * N)()
    cap = L.tnb_cp_als_factors_capacity(N, sh, R, offs)
    wsb = L.tnb_cp_als_workspace_bytes(code, N, sh, R)
    assert cap > 0 and wsb > 0
    xoff = case.get("xoff", 0)
    xbuf = torch.zeros(X64.size + xoff, dtype=dt, device="cuda")
    xbuf[xoff:] = torch.as_tensor(X64.reshape(-1)).to(dt)
    ws, pw = _guarded(wsb)
    fb = factor_byte_offset
    fbuf, pf = _guarded(fb + cap * esz)
    fac = fbuf[fb: fb + cap * esz].view(dt)
    fac.fill_(float("nan"))
    if A064 is not None:
        for n in range(N):
            fac[offs[n]: offs[n] + shape[n] * R] = torch.as_tensor(A064[n].reshape(-1)).to(dt)
    errs = (C.c_double * max(max_iter, 1))()
    iters = (C.c_int32 * 1)()
    entry = L.tnb_cp_als if A064 is None else L.tnb_cp_als_from
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(entry(code, C.c_void_p(xbuf[xoff:].data_ptr()), N, sh, R, max_iter, float("-inf"),
                     C.c_void_p(ws.data_ptr()), wsb, C.c_void_p(fac.data_ptr()), cap, errs, iters, stream))
    assert _intact(ws, wsb, pw), (case, "workspace overrun")
    assert _intact(fbuf, fb + cap * esz, pf), (case, "factors buffer overrun")
    pad = torch.ones(cap, dtype=torch.bool, device="cuda")
    for n in range(N):
        pad[offs[n]: offs[n] + shape[n] * R] = False
    assert bool(fac[pad].isnan().all()), (case, "padding between factors written")
    assert not bool(fac[~pad].isnan().any()), (case, "NaN in the factors")
    return [fac[offs[n]: offs[n] + shape[n] * R].double().cpu().numpy().reshape(shape[n], R) for n in range(N)]


CABI = {
    "n2": (CASES["n2_tc_f32"], True),
    "tree": (CASES["r64_f32"], True),
    "chfsi_start": (_case((300, 24, 20), 6, F32), False),
    "r130": (CASES["r130_f64"], True),
    "xoff": (CASES["tc_both_xoff_f32"], True),
    "tree_default_start": (CASES["small_f64"], False),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CABI))
def test_cabi_stays_inside_queried_buffers(name):
    """Workspace of exactly tnb_cp_als_workspace_bytes, factors buffer of exactly tnb_cp_als_factors_capacity: neither
    canary is touched and the padding between factors keeps its NaN; the result equals ops.cp_als."""
    from tntorch_b200 import ops

    case, given = CABI[name]
    X, A0 = _problem(case, _seed(name))
    Xd, A0d, X64, A064 = _on_device(case, X, A0)
    got = _cabi_run(case, X64, A064 if given else None, 2)
    ref = _host(ops.cp_als(Xd, case["R"], max_iter=2, tol=float("-inf"), init=A0d if given else None))
    assert all(np.array_equal(a, b) for a, b in zip(got, ref)), name


@pytest.mark.gpu
def test_misaligned_factors_match_oracle():
    """fp32 factors at a 4-byte offset with an even R: cp_khatri's 8-byte test sends every reduction to the scalar
    kernel, the projections read V element by element; the result still matches the oracle."""
    case = MISALIGNED_FACTORS
    X, A0 = _problem(case, 600)
    _, _, X64, A064 = _on_device(case, X, A0)
    orc = als_oracle(X64, A064, 1)
    kappa = max(orc["kappa"])
    assert kappa <= KAPPA_MAX, kappa
    got = _cabi_run(case, X64, A064, 1, factor_byte_offset=case["foff"])
    dev = _factor_dev(got, orc["factors"][0])
    print(f"misaligned factors: reductions {sorted({c['kernel'] for c in reductions(case, _sms())})}, "
          f"kappa {kappa:.2f}, factor dev {dev:.2e}")
    assert dev <= TOL[case["dtype"]]["factor"] * max(1.0, kappa), dev


@pytest.mark.gpu
def test_two_threads_two_streams_match_sequential():
    """Two host threads, each on its own stream, each running a different case three times: the factors are bitwise
    equal to the sequential results."""
    from tntorch_b200 import ops

    names = ["r64_f32", "wrap_f64"]
    inputs = {}
    for name in names:
        X, A0 = _problem(CASES[name], _seed(name))
        Xd, A0d, _, _ = _on_device(CASES[name], X, A0)
        inputs[name] = (Xd, A0d)
    seq = {n: ops.cp_als(inputs[n][0], CASES[n]["R"], max_iter=2, tol=float("-inf"), init=inputs[n][1]) for n in names}
    torch.cuda.synchronize()
    results, errors = {n: [] for n in names}, []

    def work(name):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for _ in range(3):
                    f = ops.cp_als(inputs[name][0], CASES[name]["R"], max_iter=2, tol=float("-inf"), init=inputs[name][1])
                    results[name].append([t.clone() for t in f])
            s.synchronize()
        except Exception as e:  # pragma: no cover - reported below
            errors.append(e)

    threads = [threading.Thread(target=work, args=(n,)) for n in names]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for n in names:
        assert len(results[n]) == 3
        for f in results[n]:
            assert all(torch.equal(a, b) for a, b in zip(f, seq[n])), n


# ==================================================================================================== sizing (CPU)
def test_factors_capacity_rejects_bad_arguments():
    from tntorch_b200 import _lib

    L = _lib.lib()
    big = (2**31 - 1) // (8 + 1)
    assert L.tnb_cp_als_factors_capacity(1, _lib.i64([5]), 2, None) == -1
    assert L.tnb_cp_als_factors_capacity(17, _lib.i64([2] * 17), 2, None) == -1
    assert L.tnb_cp_als_factors_capacity(3, _lib.i64([4, 5, 6]), 0, None) == -1
    assert L.tnb_cp_als_factors_capacity(3, _lib.i64([4, 5, 6]), 257, None) == -1
    assert L.tnb_cp_als_factors_capacity(2, _lib.i64([3, big + 1]), 8, None) == -1
    assert L.tnb_cp_als_factors_capacity(2, _lib.i64([3, big]), 8, None) > 0
    assert L.tnb_cp_als_factors_capacity(16, _lib.i64([2] * 16), 2, None) == 16 * 64
    offs = (C.c_int64 * 3)()
    assert L.tnb_cp_als_factors_capacity(3, _lib.i64([4, 17, 6]), 5, offs) == 64 + 128 + 64
    assert list(offs) == [0, 64, 192]  # each factor padded to a multiple of 64 elements


def test_workspace_bytes_refuses_16_bit_types():
    from tntorch_b200 import _lib

    L = _lib.lib()
    sh = _lib.i64([8, 7, 6])
    for code in (_lib.TNB_BF16, _lib.TNB_F16):
        assert L.tnb_cp_als_workspace_bytes(code, 3, sh, 4) == 0
    for code in (_lib.TNB_F32, _lib.TNB_F64):
        assert L.tnb_cp_als_workspace_bytes(code, 3, sh, 4) > 0
