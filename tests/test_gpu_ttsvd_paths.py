"""The dense TT-SVD path by path against a step-wise fp64 oracle.

csrc/sweep.cuh picks, per step of the right-to-left sweep, a Gram kernel (TF32 wgmma on a row-major or a K-blocked
carry, or the generic fp64-accumulating GEMM on the tall or the wide side), an eigensolver (two-sided Jacobi in fp32 or
fp64, the host-driven or the eps-only adaptive ChFSI, or the sync-free device chain), a projection (3xTF32 tensor cores
in three layouts, the FFMA kernel, the generic GEMM, or the wide factor) and whether the sweep runs speculatively.
This file
  * restates each of those choices in Python (the functions under "dispatch", each citing its C++ condition) and
    checks on the CPU that the cases below reach every choice on an SXM (132 SMs) and a PCIe (114 SMs) H100;
  * checks every step of every case against `step_oracle`, an fp64 NumPy statement that shares no code with the
    kernels or with tests/sweep_model.py.  Step mu is checked on the carry it should have seen, formed from X and the
    device's own later cores, so an error in one step does not carry into the check of the next:
      (a) the rank, (b) the captured-energy deficit of the core's row space (and, on gapped cases, its largest
      principal angle to the leading right singular vectors), (c) the gauge of cores 1..N-1, (d) the projection
      chain core_0 = X W_1^T;
    and end to end: (e) ranks and relative error against oracle.tt_oracle.tt_svd, (f) the host-driven and the
    CUDA-core-only sweeps, (g) the input unchanged, (h) two calls bitwise equal;
  * checks each case's return_info and launched kernels (torch.profiler) against the restatement, and a batch whose
    tensors are partly accepted and partly repeated against their single calls.
Run with -s to see the measured deviations and paths."""
import numpy as np
import pytest
import torch

from oracle import cases as ocases
from oracle import tt_oracle as orc

F32, F64 = torch.float32, torch.float64
BF16, F16, E4M3 = torch.bfloat16, torch.float16, torch.float8_e4m3fn
LOW = (BF16, F16, E4M3)
ESZ = {F64: 8, F32: 4, BF16: 2, F16: 2, E4M3: 1}

# Bounds, per compute type (a 16-bit or fp8 input computes in fp32).  rank: none, exact; subspace: (b) captured-energy
# deficit / ||C_mu||^2; angle: (b) sin of the largest principal angle on gapped cases; gauge: (c); chain: (d); relerr:
# (e) and (f) |relerr - oracle relerr|.  Each is at most 10x the largest value measured on an H100 SXM (132 SMs, 700 W)
# over the cases here, printed with -s:
#   fp64: subspace 7.8e-13, angle 3.8e-6, relerr 6.2e-11 (L257_f64: the host ChFSI's 1e-6 stop), gauge 9.2e-14,
#         chain 5.9e-14 (L64_f64);
#   fp32: subspace 1.2e-8 and angle 6.2e-4 (L512_cap64_f32: the sync-free chain), gauge 3.7e-7 (L112_f32), chain 1.1e-6
#         (kblocked_r16_f32), relerr 1.8e-7 (cap_above_f32).
TOL = {
    F64: dict(subspace=7.8e-12, angle=3.8e-5, gauge=9e-13, chain=5.9e-13, relerr=6.2e-10),
    F32: dict(subspace=1.2e-7, angle=6e-3, gauge=3.7e-6, chain=1.1e-5, relerr=1.8e-6),
}


# ==================================================================================================== fp64 oracle
def right_interface(cores, mu):
    """W (r_mu x I_mu...I_{N-1}): cores mu..N-1 contracted, fp64."""
    W = np.ones((1, 1))
    for c in reversed(cores[mu:]):
        r0, I, r1 = c.shape
        W = (c.reshape(r0 * I, r1) @ W).reshape(r0, -1)
    return W


def rank_rule(lam, delta2, cap):
    """round.py:147-158 on descending squared singular values."""
    lam = np.maximum(np.asarray(lam, dtype=np.float64), 0.0)
    tail = np.cumsum(lam[::-1])
    drop = int(np.sum(tail <= delta2))
    return max(1, min(cap, len(lam) - drop))


def step_oracle(X, cores, eps, caps, gram_class):
    """Per step mu = N-1..1, against the carry C_mu = X_(<=mu) W_{mu+1}^T made from the device's later cores:
    rank, captured-energy deficit, principal angle (sin) to V_r, gauge deviation; then the chain deviation of core 0.
    gram_class: the expected ranks follow the eigenvalues of the fp64 Gram (DESIGN.md section 6, exactly rank-deficient
    data) instead of the SVD."""
    X = np.asarray(X, dtype=np.float64)
    N = X.ndim
    shape = X.shape
    nx2 = float(np.vdot(X, X))
    delta2 = (eps / max(1.0, np.sqrt(N - 1))) ** 2 * nx2
    out = []
    for mu in range(N - 1, 0, -1):
        W = right_interface(cores, mu + 1)
        rows = int(np.prod(shape[:mu]))
        C = (X.reshape(rows * shape[mu], -1) @ W.T).reshape(rows, -1)
        sv = np.linalg.svd(C, compute_uv=False) if min(C.shape) else np.zeros(0)
        if gram_class:
            G = C @ C.T if C.shape[0] <= C.shape[1] else C.T @ C
            lam = np.sort(np.linalg.eigvalsh(G))[::-1]
        else:
            lam = sv ** 2
        cap = min(caps[mu - 1] or 1 << 30, *C.shape)
        want = rank_rule(lam, delta2, cap) if sv.size and sv[0] >= 1e-13 else 1
        M = cores[mu].reshape(cores[mu].shape[0], -1)
        r = M.shape[0]
        c2 = float(np.vdot(C, C))
        Q = np.linalg.qr(M.T)[0]
        deficit = (float(np.sum(sv[:r] ** 2)) - float(np.linalg.norm(C @ Q) ** 2)) / c2 if c2 > 0 else 0.0
        angle = None
        if c2 > 0 and r < len(sv) and sv[r] < 0.5 * sv[r - 1] and sv[r - 1] - sv[r] >= 1e-2 * sv[0]:
            Vr = np.linalg.svd(C, full_matrices=False)[2][:r].T
            angle = float(np.linalg.norm(Vr - Q @ (Q.T @ Vr), 2))
        gauge = float(np.abs(M @ M.T - np.eye(r)).max())
        out.append(dict(mu=mu, rank=r, want=want, deficit=deficit, angle=angle, gauge=gauge))
    W1 = right_interface(cores, 1)
    core0 = cores[0].reshape(shape[0], -1)
    chain = float(np.linalg.norm(core0 - X.reshape(shape[0], -1) @ W1.T) / np.sqrt(nx2)) if nx2 > 0 else 0.0
    return out, chain


# ==================================================================================================== dispatch
# One function per device choice; `sms` is cudaDevAttrMultiProcessorCount (device_info().sm_count).
TC_MIN_ROWS = 2048  # sweep.cuh: TC_MIN_ROWS
PROJ_TC_MIN_ROWS = 16384  # sweep.cuh: PROJ_TC_MIN_ROWS
JACOBI_MAX_N = 256  # jacobi.cuh: JACOBI_MAX_N
JAC2_MAX_N_F64, JAC2_MAX_N_F32, JAC2_MIXED_MAX_N = 80, 112, 64  # jacobi2.cuh
PT_MAX_N = 64  # project_tc.cuh: PT_MAX_N
CD_MAX_B = 96  # chfsi_dev.cuh: CD_MAX_B
CF_KS = 8  # cheb_filter.cuh: CF_KS


def compute_type(dtype):
    return F64 if dtype == F64 else F32


def gram_tc_input_ok(dtype, rows, n):
    """gram_tc.cuh gram_tc_input_ok: fp32 gram_tc_shape_ok (16 <= n <= 16384, n % 4 == 0, rows < 2^31 - 64); bf16 /
    fp16 also n % 8 == 0 and (a fold > 1, n == 128 or n >= 256); fp8 also n % 16 == 0; fp64 never."""
    if dtype == F64:
        return False
    ok = n >= 16 and n % 4 == 0 and n <= 16384 and 1 <= rows < (1 << 31) - 64
    if dtype == F32:
        return ok
    fold = 1 if (n >= 128 or n < 32 or 128 % n) else (128 // n if rows % (128 // n) == 0 else 1)
    ok = ok and n % 8 == 0 and (fold > 1 or n == 128 or n >= 256)
    return ok and (n % 16 == 0 if dtype == E4M3 else True)


def project_tc_shape_ok(dtype, rows, K, r, aligned):
    """project_tc.cuh project_tc_shape_ok: 1 <= r <= 64, K a multiple of 16 bytes, K >= 128 bytes (64 for fp8),
    K <= 2^24, 128 <= rows < 2^31 - 256, A and C 16-byte aligned."""
    esz = ESZ[dtype]
    kmin = 64 if esz == 1 else 128 // esz
    return (1 <= r <= PT_MAX_N and K % (16 // esz) == 0 and kmin <= K <= 1 << 24 and 128 <= rows < (1 << 31) - 256
            and aligned)


def project_use_tc(dtype, rows, n, r, aligned):
    """sweep.cuh project_use_tc: a tensor-core input type (not fp64), rows >= PROJ_TC_MIN_ROWS, project_tc_shape_ok."""
    return dtype != F64 and rows >= PROJ_TC_MIN_ROWS and project_tc_shape_ok(dtype, rows, n, r, aligned)


def project_kernel(dtype, rows, n, r, kcap, aligned):
    """sweep.cuh project_any with the workspace of project_tc_carve_bytes (sized at kcap, pointers aligned):
    tc, else ffma for fp32 input (project.cuh project_f32_fast_ok: 1 <= r <= 64, n % 4 == 0, n >= 4, aligned), else
    the generic GEMM."""
    ws = dtype != F64 and rows >= n and project_use_tc(dtype, rows, n, kcap, True)
    if ws and project_use_tc(dtype, rows, n, r, aligned):
        return "tc"
    if dtype == F32 and 1 <= r <= 64 and n % 4 == 0 and n >= 4 and aligned:
        return "ffma"
    return "generic"


def dims(shape, rmax):
    """sweep.cuh make_dims: rows[mu] = prod_{j<mu} I_j; rcap[mu] = min(I_mu rcap[mu+1], rows[mu], rmax)."""
    N = len(shape)
    rows = [1] * (N + 1)
    for k in range(N):
        rows[k + 1] = rows[k] * shape[k]
    rcap = [1] * (N + 1)
    for mu in range(N - 1, 0, -1):
        c = min(shape[mu] * rcap[mu + 1], rows[mu])
        if rmax and rmax[mu - 1]:
            c = min(c, rmax[mu - 1])
        rcap[mu] = c
    return rows, rcap


def carry_kblocked(dtype, shape, rcap, rows, mu, aligned):
    """sweep.cuh carry_kblocked: fp32 compute, reader step mu tall with rows >= 16384, gram_tc_kblocked_shape_ok
    (n >= 256, n % 8 == 0, rows % 8 == 0) and a tensor-core projection at min(rcap, n) <= 64; writer step mu + 1 tall,
    n >= 32, projecting on the tensor cores, rcap[mu+1] % 16 == 0 and <= 48, I_mu % 16 == 0, and, when it is step 0,
    a 16-byte aligned input; and the carry the writer reads is not K-blocked itself."""
    N = len(shape)
    if compute_type(dtype) != F32 or mu < 1 or mu + 1 > N - 1:
        return False
    r_, n = rows[mu], shape[mu] * rcap[mu + 1]
    k = min(rcap[mu], n)
    reader = (r_ >= n and r_ >= PROJ_TC_MIN_ROWS and gram_tc_input_ok(F32, r_, n) and n >= 256 and n % 8 == 0
              and r_ % 8 == 0 and k <= PT_MAX_N and project_tc_shape_ok(F32, r_, n, k, True))
    first = mu + 1 == N - 1
    wr, wn, r = rows[mu + 1], shape[mu + 1] * rcap[mu + 2], rcap[mu + 1]
    wtc = project_use_tc(dtype if first else F32, wr, wn, r, True)
    writer = (wr >= wn and wn >= 32 and wtc and r % 16 == 0 and r <= 48 and shape[mu] % 16 == 0
              and (not first or aligned))
    return reader and writer and not carry_kblocked(dtype, shape, rcap, rows, mu + 1, aligned)


def chfsi_dev_block(L, k):
    """chfsi_dev.cuh chfsi_dev_block."""
    g = max(k // 2, 16)
    b = (k + g + 3) // 4 * 4
    return L // 4 * 4 if b > L else b


def cheb_filter_shape_ok(L, b, sms):
    """cheb_filter.cuh cheb_filter_shape_ok: L % 256 == 0, 8 <= b <= 128, b % 4 == 0, (L / 128) * CF_KS <= SMs and
    the shared memory of cheb_filter_smem_bytes within 227 KB."""
    if L % 256 or L < 256 or b < 8 or b % 4 or b > 128 or (L // 128) * CF_KS > sms:
        return False
    nbox, ksl = (b + 31) // 32, L // CF_KS
    return ksl * 128 * 4 + ksl * nbox * 128 + nbox * 32 * 129 * 4 + 1088 <= 227 * 1024


def spec_step_ok(dtype, rows, n, cap, sms):
    """sweep.cuh spec_step_ok: a Gram side L <= 256, or fp32 with k = min(cap, L), k + 16 <= 256 and chfsi_dev_ok
    (chfsi_dev.cuh: 8 <= b <= CD_MAX_B, b % 4 == 0, cheb_filter_shape_ok, b <= JAC2_MAX_N_F32)."""
    L = min(rows, n)
    if L <= JACOBI_MAX_N:
        return True
    if compute_type(dtype) != F32:
        return False
    k = min(cap, L)
    if k + 16 > JACOBI_MAX_N:
        return False
    b = chfsi_dev_block(L, k)
    return 8 <= b <= CD_MAX_B and b % 4 == 0 and cheb_filter_shape_ok(L, b, sms) and b <= JAC2_MAX_N_F32


def speculative(case, sms):
    """sweep.cuh spec_eligible: N >= 2, a cap on every bond, (eps / sqrt(N-1))^2 < 1e-20, every step spec_step_ok."""
    shape, rmax, eps = case["shape"], case["rmax"], case["eps"]
    N = len(shape)
    if N < 2 or not rmax or not all(rmax) or not (eps / max(1.0, np.sqrt(N - 1))) ** 2 < 1e-20:
        return False
    rows, rcap = dims(shape, rmax)
    return all(spec_step_ok(case["dtype"], rows[mu], shape[mu] * rcap[mu + 1], rcap[mu], sms) for mu in range(N - 1, 0, -1))


def eig_kernel(dtype, L, spec, exact, have_rmax):
    """Speculative (spec_step_eig_begin): L <= 256 -> jacobi2_eigh with fp32 rotations for fp32 compute on the tensor-core
    sweep when L <= JAC2_MAX_N_F32, else fp64; L > 256 -> the sync-free chain (cd_*).  Host-driven (eig_carve /
    eig_run): jacobi2_eigh in fp64 for L <= 256, else the host ChFSI (adaptive without a cap).  jacobi2_eigh
    (jacobi2.cuh): fp64 8 <= L <= 64 the mixed kernel, L <= 80 jacobi2 fp64, above that jacobi_eigh."""
    if L > JACOBI_MAX_N:
        return "cd" if spec else ("chfsi" if have_rmax else "chfsi_adaptive")
    if spec and compute_type(dtype) == F32 and not exact and L <= JAC2_MAX_N_F32:
        return "jacobi2_f32"
    if 8 <= L <= JAC2_MIXED_MAX_N:
        return "jacobi2_mixed"
    return "jacobi2_f64" if L <= JAC2_MAX_N_F64 else "jacobi_f64"


def steps(case, sms, spec=None, ranks=None, exact=False):
    """Per step mu = N-1..1: dict(mu, rows, n, L, gram, eig, proj).  spec None: as the dispatcher decides; ranks: the
    ranks of a host-driven sweep (its n follows the chosen rank, not the cap); exact: a TF32 rejection's repeat.
    gram (gram_small_side / spec_step_gram): tc_kblocked when the carry is K-blocked; tc on the tall side with rows >=
    TC_MIN_ROWS, gram_tc_input_ok, the tensor-core sweep and, at step 0, an aligned input; generic_tall / generic_wide
    otherwise.  proj (step_factors): wide; tc_in_kb / tc_out_kb on a K-blocked carry; else project_kernel."""
    shape, rmax, dtype = case["shape"], case["rmax"], case["dtype"]
    N = len(shape)
    spec = speculative(case, sms) if spec is None else spec
    tc = case.get("tc", True)
    rows_, rcap = dims(shape, rmax)
    aligned = case.get("off", 0) * ESZ[dtype] % 16 == 0
    eps2 = (case["eps"] / max(1.0, np.sqrt(N - 1))) ** 2
    tc_gram = tc and not exact and (spec or eps2 < 1e-20 or eps2 >= 1e-4)
    out = []
    for mu in range(N - 1, 0, -1):
        first = mu == N - 1
        rn = rcap[mu + 1] if spec or ranks is None else ranks[mu + 1]
        rows, n = rows_[mu], shape[mu] * rn
        L = min(rows, n)
        din = dtype if first else compute_type(dtype)
        kin = spec and tc and carry_kblocked(dtype, shape, rcap, rows_, mu, aligned)
        kout = spec and tc and carry_kblocked(dtype, shape, rcap, rows_, mu - 1, aligned)
        al = aligned or not first
        if kin:
            gram = "tc_kblocked"
        elif rows >= n and tc_gram and rows >= TC_MIN_ROWS and gram_tc_input_ok(din, rows, n) and al:
            gram = "tc"
        else:
            gram = "generic_tall" if rows >= n else "generic_wide"
        kcap = min(rcap[mu], L)
        r = kcap if spec or ranks is None else ranks[mu]
        if rows < n:
            proj = "wide"
        elif kin:
            proj = "tc_in_kb"
        elif kout:
            proj = "tc_out_kb"
        else:
            proj = project_kernel(din, rows, n, r, kcap, al) if tc else (
                "ffma" if din == F32 and 1 <= r <= 64 and n % 4 == 0 and al else "generic")
        eig = eig_kernel(dtype, L, spec, exact or not tc, bool(rmax and rmax[mu - 1]))
        out.append(dict(mu=mu, rows=rows, n=n, L=L, gram=gram, eig=eig, proj=proj))
    return out


def expected_flags(case, want_ranks):
    """spec_check_kernel bits of an eligible case: 0 the TF32 / fp32-solve noise floor rejects the spectrum (marked on
    the case, it depends on the data), 4 a rank below the cap, 5 a zero unfolding."""
    rows, rcap = dims(case["shape"], case["rmax"])
    f = 1 if case.get("reject") else 0
    if any(want_ranks[mu] != rcap[mu] for mu in range(1, len(case["shape"]))):
        f |= 16
    if case["kind"] == "zero":
        f |= 32
    return f


# ==================================================================================================== cases
def _case(shape, rmax, dtype, kind="tt", eps=1e-14, **kw):
    if rmax is not None and not hasattr(rmax, "__len__"):
        rmax = [rmax] * (len(shape) - 1)
    return dict(shape=tuple(shape), rmax=rmax, dtype=dtype, kind=kind, eps=eps, **kw)


CASES = {
    # K-blocked carry: step 0 writes the carry step 1 reads
    "kblocked_r16_f32": _case((128, 128, 16, 32), 16, F32),
    "kblocked_r48_f32": _case((128, 128, 16, 64), 48, F32, reject=True),
    # TF32 Gram thresholds: rows 2047 / 2048, n % 4 != 0, n = 16
    "rows2047_f32": _case((23, 89, 32), 8, F32),
    "rows2048_f32": _case((32, 64, 32), 8, F32),
    "rows2048_f64": _case((32, 64, 32), 8, F64),
    "n18_f32": _case((64, 64, 18), 8, F32),
    "n16_f32": _case((64, 64, 16), 8, F32),
    # projection thresholds: rows 16383 / 16384
    "rows16383_f32": _case((127, 129, 32), 8, F32),
    "rows16384_f32": _case((128, 128, 32), 8, F32),
    "rows16384_f64": _case((128, 128, 32), 8, F64),
    # eigensolver boundaries
    "L64_f64": _case((40, 60, 64), 12, F64),
    "L80_f64": _case((40, 60, 80), 12, F64),
    "L81_f64": _case((40, 60, 81), 12, F64),
    "L112_f32": _case((40, 60, 112), 12, F32),
    "L113_f32": _case((40, 60, 113), 12, F32),
    "L256_f32": _case((16, 32, 256), 12, F32),
    "L257_f32": _case((16, 32, 257), 12, F32),
    "L257_f64": _case((16, 32, 257), 12, F64),
    "L512_cap64_f32": _case((8, 64, 512), 64, F32),
    "L512_cap65_f32": _case((8, 64, 512), 65, F32),
    "L2048_cap32_f32": _case((4, 512, 2048), 32, F32),
    # eps-only: k grows 32 -> 64 -> 128
    "eps_only_f32": _case((16, 32, 512), None, F32, kind="geometric", eps=1e-2, q=0.93),
    "eps_only_f64": _case((16, 32, 512), None, F64, kind="geometric", eps=1e-3, q=0.93),
    # wide steps
    "wide_first_f32": _case((8, 300), 6, F32),
    "wide_first_f64": _case((8, 300), 6, F64),
    "wide_middle_f32": _case((6, 10, 40, 8), 12, F32),
    "wide_middle_f64": _case((6, 10, 40, 8), 12, F64),
    "smooth_f32_r6": _case((20, 18, 16, 14), 6, F32, kind="golden", reject=True),
    "wide_below_cap_f32": _case((4, 8, 64), 16, F32, kind="exact", rank=2, reject=True),
    "wide_below_cap_f64": _case((4, 8, 64), 16, F64, kind="exact", rank=2),
    # small and degenerate shapes
    "n1_f32": _case((37,), None, F32, kind="randn"),
    "n2_f64": _case((30, 20), 5, F64),
    "unit_front_f32": _case((1, 12, 10, 8), 4, F32),
    "unit_middle_f64": _case((12, 1, 10, 8), 4, F64),
    "unit_end_f32": _case((12, 10, 8, 1), 4, F32),
    "rmax1_f64": _case((10, 12, 14), 1, F64),
    "cap_above_f32": _case((5, 6, 7), 50, F32, kind="randn"),
    # misaligned input: a TF32-eligible step 0, and step 0 as the K-blocked writer
    "offset_tc_f32": _case((64, 64, 32), 8, F32, off=1),
    "offset_kblocked_f32": _case((128, 128, 16, 32), 16, F32, off=1),
    # fallbacks
    "lownoise_f32": _case((32, 64, 32), 4, F32, kind="tt", noise=1e-7, reject=True),
    "slice_f32": _case((12, 10, 8), 4, F32, kind="slice", reject=True),
    "slice_f64": _case((12, 10, 8), 4, F64, kind="slice"),
    "zero_f32": _case((12, 10, 8), 4, F32, kind="zero"),
    # CUDA cores only
    "no_tc_f32": _case((128, 128, 32), 8, F32, tc=False),
    # other input types: a wide step, and an offset with a tensor-core-eligible step 0 (gauge and alignment only)
    "wide_bf16": _case((8, 16, 256), 16, BF16),
    "offset_bf16": _case((64, 64, 128), 8, BF16, off=1),
    "wide_f16": _case((8, 16, 256), 16, F16),
    "offset_f16": _case((64, 64, 128), 8, F16, off=1),
    "wide_e4m3": _case((8, 16, 256), 16, E4M3),
    "offset_e4m3": _case((64, 64, 128), 8, E4M3, off=1),
}
# eps-only at a rank the subspace eigensolver cannot reach (> 240): refused
RANK241 = _case((16, 32, 512), None, F32, kind="geometric", eps=1e-3, q=0.995)


def _coverage(sms):
    seen = set()
    for c in CASES.values():
        if len(c["shape"]) < 2:
            seen.add(("N", 1))
            continue
        spec = speculative(c, sms)
        seen.add(("spec", spec))
        for s in steps(c, sms):
            seen |= {("gram", s["gram"]), ("eig", s["eig"]), ("proj", s["proj"])}
        if not spec:  # a host-driven sweep at the caps (the rank rule decides the rest)
            for s in steps(c, sms, spec=False):
                seen |= {("gram", s["gram"]), ("eig", s["eig"]), ("proj", s["proj"])}
        if spec and c.get("reject"):
            seen.add(("flag", 0))
        if spec and c["kind"] in ("slice", "exact"):
            seen.add(("flag", 4))
        if spec and c["kind"] == "zero":
            seen.add(("flag", 5))
        if c.get("off") and c["dtype"] == F32:  # what step 0 would run on an aligned copy
            rows, rcap = dims(c["shape"], c["rmax"])
            kb = carry_kblocked(F32, c["shape"], rcap, rows, len(c["shape"]) - 2, True)
            seen.add(("offset", "kblocked" if kb else steps(dict(c, off=0), sms)[0]["gram"]))
    return seen


@pytest.mark.parametrize("sms", [132, 114])
def test_cases_cover_every_dispatch_choice(sms):
    """CPU: the case list reaches every Gram kernel, eigensolver and projection, both control paths and every flag an
    input can raise honestly, on an SXM and a PCIe H100 (L = 2048 runs the sync-free chain on 132 SMs only; the
    114-SM card still reaches it at L = 512)."""
    seen = _coverage(sms)
    want = {("gram", g) for g in ("tc", "tc_kblocked", "generic_tall", "generic_wide")}
    want |= {("eig", e) for e in ("jacobi2_f32", "jacobi2_mixed", "jacobi2_f64", "jacobi_f64", "cd", "chfsi",
                                   "chfsi_adaptive")}
    want |= {("proj", p) for p in ("tc", "tc_in_kb", "tc_out_kb", "ffma", "generic", "wide")}
    want |= {("spec", True), ("spec", False), ("flag", 0), ("flag", 4), ("flag", 5), ("N", 1)}
    want |= {("offset", "kblocked"), ("offset", "tc")}
    assert not want - seen, sorted(want - seen)


def test_dispatch_restatement_spot_checks():
    """CPU: the restatement gives what the case names claim."""
    for sms in (132, 114):
        s = steps(CASES["kblocked_r16_f32"], sms)
        assert [x["gram"] for x in s] == ["tc", "tc_kblocked", "generic_wide"]
        assert [x["proj"] for x in s] == ["tc_out_kb", "tc_in_kb", "wide"]
        s = steps(CASES["offset_kblocked_f32"], sms)
        assert [x["gram"] for x in s] == ["generic_tall", "tc", "generic_wide"]
        assert [x["proj"] for x in s] == ["generic", "tc", "wide"]
        assert steps(CASES["offset_tc_f32"], sms)[0]["gram"] == "generic_tall"
        assert steps(CASES["rows2047_f32"], sms)[0]["gram"] == "generic_tall"
        assert steps(CASES["rows2048_f32"], sms)[0]["gram"] == "tc"
        assert steps(CASES["rows2048_f64"], sms)[0]["gram"] == "generic_tall"
        assert steps(CASES["n18_f32"], sms)[0]["gram"] == "generic_tall"
        assert steps(CASES["n16_f32"], sms)[0]["gram"] == "tc"
        assert steps(CASES["rows16383_f32"], sms)[0]["proj"] == "ffma"
        assert steps(CASES["rows16384_f32"], sms)[0]["proj"] == "tc"
        assert steps(CASES["no_tc_f32"], sms)[0]["proj"] == "ffma"
        assert [steps(CASES[k], sms)[0]["eig"] for k in ("L64_f64", "L80_f64", "L81_f64", "L112_f32", "L113_f32",
                                                          "L256_f32")] == [
            "jacobi2_mixed", "jacobi2_f64", "jacobi_f64", "jacobi2_f32", "jacobi_f64", "jacobi_f64"]
        assert not speculative(CASES["L257_f32"], sms) and steps(CASES["L257_f32"], sms)[0]["eig"] == "chfsi"
        assert speculative(CASES["L512_cap64_f32"], sms) and steps(CASES["L512_cap64_f32"], sms)[0]["eig"] == "cd"
        assert not speculative(CASES["L512_cap65_f32"], sms)
        assert steps(CASES["eps_only_f32"], sms)[0]["eig"] == "chfsi_adaptive"
        assert [x["proj"] for x in steps(CASES["wide_middle_f32"], sms)] == ["ffma", "wide", "wide"]
    assert speculative(CASES["L2048_cap32_f32"], 132) and not speculative(CASES["L2048_cap32_f32"], 114)
    assert steps(CASES["L2048_cap32_f32"], 132)[0]["eig"] == "cd"
    assert steps(CASES["L2048_cap32_f32"], 114)[0]["eig"] == "chfsi"


# ==================================================================================================== inputs
def _seed(name):
    return sum(ord(c) * (i + 1) for i, c in enumerate(name)) % 10007


def _random_tt(shape, rank, rng):
    """The full tensor of a TT with Gaussian cores and ranks min(rank, the unfolding's sides)."""
    N = len(shape)
    ranks = [1] + [min(rank, int(np.prod(shape[:k])), int(np.prod(shape[k:]))) for k in range(1, N)] + [1]
    X = np.ones((1, 1))
    for k in range(N):
        X = (X @ rng.standard_normal((ranks[k], shape[k] * ranks[k + 1]))).reshape(-1, ranks[k + 1])
    return X.reshape(shape)


def make_input(case, seed):
    """fp64 NumPy data of the case."""
    rng = np.random.default_rng(seed)
    shape, kind = case["shape"], case["kind"]
    if kind == "randn":
        return rng.standard_normal(shape)
    if kind == "zero":
        return np.zeros(shape)
    if kind == "golden":
        return ocases.make_dense(ocases.TTSVD_CASES["smooth_f32_r6"]).astype(np.float64)
    if kind == "geometric":  # a (rows x last) matrix with singular values q^i, reshaped
        m = int(np.prod(shape[:-1]))
        k = min(m, shape[-1])
        U = np.linalg.qr(rng.standard_normal((m, k)))[0]
        V = np.linalg.qr(rng.standard_normal((shape[-1], k)))[0]
        return ((U * case["q"] ** np.arange(k)) @ V.T).reshape(shape)
    if kind == "slice":
        X = np.zeros(shape)
        X[..., 0] = rng.standard_normal(shape[:-1])
        return X
    if kind == "exact":
        return _random_tt(shape, case["rank"], rng)
    rank = max(case["rmax"] or [1]) if case["rmax"] else 4
    X = _random_tt(shape, rank, rng)
    noise = case.get("noise", 0.3)
    return X + noise * np.linalg.norm(X) / np.sqrt(X.size) * rng.standard_normal(shape)


def on_device(case, X):
    """(device tensor in the case's dtype, at `off` elements past an aligned address; its values as fp64 NumPy)."""
    dt, off = case["dtype"], case.get("off", 0)
    t = torch.as_tensor(X).to(dt)
    if off:
        buf = torch.zeros(t.numel() + off, dtype=dt)
        buf[off:] = t.reshape(-1)
        d = buf.cuda()[off:].view(t.shape)
        assert d.is_contiguous() and d.data_ptr() % 16 == off * ESZ[dt] % 16
    else:
        d = t.cuda()
    return d, d.cpu().to(torch.float64).numpy()


def host(cores):
    return [c.detach().cpu().to(torch.float64).numpy() for c in cores]


def ranks_of(cores):
    return [1] + [int(c.shape[2]) for c in cores]


def relerr(X64, cores):
    return orc.relative_error(X64, cores)


def _sms():
    from tntorch_b200 import ops

    ops.set_reserved_sms(0)
    return torch.cuda.get_device_properties(0).multi_processor_count


def _run(d, case, **kw):
    from tntorch_b200 import ops

    tc = kw.pop("use_tensorcore", True) and case.get("tc", True)
    return ops.ttsvd(d, rmax=case["rmax"], eps=case["eps"], return_info=True, use_tensorcore=tc, **kw)


# ==================================================================================================== per step
GPU_CASES = [n for n, c in CASES.items() if c["dtype"] in (F32, F64)]


@pytest.mark.gpu
@pytest.mark.parametrize("name", GPU_CASES)
def test_steps_match_oracle(name):
    """(a)-(h) for one case; also return_info against the restatement.  Exactly rank-deficient cases (kind "exact")
    check no rank: the tail rule chooses among directions at the Gram's rounding level, which no oracle reproduces
    (DESIGN.md section 6), so (a) and the rank half of (e) are skipped and the expected flags follow the device's ranks;
    what they check is that the rows kept at that level are orthonormal (c) and the rest of (b)-(h)."""
    case = CASES[name]
    sms = _sms()
    dt = case["dtype"]
    tol = TOL[compute_type(dt)]
    X = make_input(case, _seed(name))
    d, X64 = on_device(case, X)
    before = d.clone()
    cores, info = _run(d, case)
    again, _ = _run(d, case)
    torch.cuda.synchronize()
    C = host(cores)
    N = len(case["shape"])
    gram_class = case["kind"] in ("exact", "slice")
    per, chain = step_oracle(X64, C, case["eps"], case["rmax"] or [0] * max(N - 1, 0), gram_class)
    spec = speculative(case, sms)
    want_ranks = [1] + [s["want"] for s in reversed(per)] + [1] if N > 1 else [1, 1]
    if case["kind"] == "exact":
        # the null space of exactly rank-deficient data sits at the Gram's rounding level: which of its directions the
        # tail rule keeps is not reproducible (DESIGN.md section 6); the kept rows must still be orthonormal
        want_ranks = ranks_of(cores)
    flags = expected_flags(case, want_ranks) if spec else 0
    accepted = spec and flags == 0
    path = steps(case, sms, spec=accepted, ranks=want_ranks, exact=bool(flags & 1))
    fmt = lambda v: "-" if v is None else f"{v:.1e}"  # noqa: E731
    print(f"\n{name}: sms {sms}, speculative {spec} flags {info['spec_flags']} (want {flags}), ranks {ranks_of(cores)}")
    for s, p in zip(per, path):
        print(f"  mu {s['mu']}: {p['rows']}x{p['n']} gram {p['gram']} eig {p['eig']} proj {p['proj']}; rank {s['rank']} "
              f"(oracle {s['want']}), deficit {s['deficit']:.1e}, angle {fmt(s['angle'])}, gauge {s['gauge']:.1e}")
    print(f"  chain {chain:.1e}")
    # (a)-(d)
    assert ranks_of(cores) == want_ranks, (name, ranks_of(cores), want_ranks)
    for s in per:
        assert s["deficit"] <= tol["subspace"], (name, s)
        assert s["angle"] is None or s["angle"] <= tol["angle"], (name, s)
        # a zero tensor has zero cores (round.py:137-145), no gauge
        assert case["kind"] == "zero" or s["gauge"] <= tol["gauge"], (name, s)
    assert chain <= tol["chain"], (name, chain)
    # return_info against the restatement
    assert info["speculative"] == int(accepted) and info["spec_flags"] == flags, (name, info, flags)
    if accepted:
        assert info["kblocked_steps"] == sum(p["gram"] == "tc_kblocked" for p in path), (name, info)
        assert info["tc_grams"] == sum(p["gram"].startswith("tc") for p in path), (name, info)
        assert (info["fused_filters"] > 0) == any(p["eig"] == "cd" for p in path), (name, info)
    elif not (flags & 1) and not case.get("reject"):
        assert info["kblocked_steps"] == 0 and info["tc_grams"] == sum(p["gram"] == "tc" for p in path), (name, info)
    else:
        assert info["tc_grams"] == 0, (name, info)
    # (e) end to end against the reference's algorithm
    ref = orc.tt_svd(X64, ranks_tt=case["rmax"], eps=None if case["rmax"] else case["eps"],
                     algorithm="eig" if gram_class else "svd")
    e_lib, e_ref = relerr(X64, C), relerr(X64, ref)
    print(f"  relerr {e_lib:.8e}, oracle {e_ref:.8e}, |diff| {abs(e_lib - e_ref):.1e}")
    if case["kind"] != "exact":
        assert ranks_of(cores) == ranks_of(ref), (name, ranks_of(ref))
    assert case["kind"] == "zero" or abs(e_lib - e_ref) <= tol["relerr"], (name, e_lib, e_ref)
    # (f) the host-driven and the CUDA-core-only sweeps
    for kw in (dict(speculate=False), dict(use_tensorcore=False)):
        other, oinfo = _run(d, case, **kw)
        e_o = relerr(X64, host(other))
        print(f"  {kw}: relerr |diff| {abs(e_o - e_lib):.1e}, tc_grams {oinfo['tc_grams']}")
        assert case["kind"] == "exact" or ranks_of(other) == ranks_of(cores), (name, kw)
        assert case["kind"] == "zero" or abs(e_o - e_lib) <= tol["relerr"], (name, kw, e_o, e_lib)
        ntc = sum(p["gram"] == "tc" for p in steps(case, sms, spec=False))
        if case.get("reject") and "speculate" in kw and ntc:
            # the host-driven sweep repeats a rejected TF32 step on the exact Gram (truncate_step)
            assert oinfo["tc_grams"] < ntc and oinfo["speculative"] == 0, (name, kw, oinfo)
    # (g), (h)
    assert torch.equal(d, before), "input modified"
    assert all(torch.equal(a, b) for a, b in zip(cores, again)), "cores not deterministic"


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c["dtype"] in LOW])
def test_low_precision_input_gauge_and_alignment(name):
    """bf16 / fp16 / e4m3 input: a wide step and a 2- or 1-byte offset run, and cores 1..N-1 are orthonormal (their
    accuracy is covered by test_gpu_bf16.py, test_gpu_fp16.py and test_gpu_fp8.py)."""
    case = CASES[name]
    sms = _sms()
    X = make_input(case, _seed(name))
    d, X64 = on_device(case, X)
    before = d.clone()
    cores, info = _run(d, case)
    C = host(cores)
    per, chain = step_oracle(X64, C, case["eps"], case["rmax"], False)
    path = steps(case, sms)
    print(f"\n{name}: speculative {info['speculative']} flags {info['spec_flags']}, path "
          f"{[(p['gram'], p['proj']) for p in path]}, gauge {[f'{s['gauge']:.1e}' for s in per]}, chain {chain:.1e}")
    assert torch.equal(d, before)
    for s in per:
        assert s["gauge"] <= TOL[F32]["gauge"], (name, s)
    assert chain <= TOL[F32]["chain"], (name, chain)


@pytest.mark.gpu
def test_rank_above_240_is_refused():
    """eps-only truncation of a Gram side above 256 whose rank passes 240 raises (the subspace eigensolver's limit)."""
    X = make_input(RANK241, 7)
    d, _ = on_device(RANK241, X)
    with pytest.raises(NotImplementedError):
        _run(d, RANK241)


# ==================================================================================================== kernels
_KERNELS = {
    "gram_tc_kernel": "gram_tc", "project_tc_kernel": "project_tc", "project_f32_kernel": "project_f32",
    "jacobi2_eigh_kernel<float>": "jacobi2_f32", "jacobi2_eigh_kernel<double>": "jacobi2_f64",
    "jacobi2_mixed_kernel": "jacobi2_mixed", "jacobi_eigh_kernel<double": "jacobi_f64", "cd_rr_kernel": "cd",
    "cheb_filter_kernel": "cheb_filter", "wide_apply_kernel": "wide",
}
_GRAM = {"tc": "gram_tc", "tc_kblocked": "gram_tc"}
_PROJ = {"tc": "project_tc", "tc_in_kb": "project_tc", "tc_out_kb": "project_tc", "ffma": "project_f32",
         "wide": "wide"}


def _want_kernels(path):
    want = set()
    for p in path:
        want |= {_GRAM.get(p["gram"]), _PROJ.get(p["proj"])}
        want |= {"cd", "cheb_filter"} if p["eig"] == "cd" else {p["eig"]}
    return want - {None}


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in GPU_CASES if len(CASES[n]["shape"]) > 1 and CASES[n]["kind"] not in (
    "slice", "zero", "exact") and not CASES[n].get("reject") and CASES[n]["rmax"]])
def test_launched_kernels_match_restatement(name):
    """The kernels one call launches (torch.profiler) are the ones the restatement names."""
    from torch.profiler import ProfilerActivity, profile

    case = CASES[name]
    sms = _sms()
    d, _ = on_device(case, make_input(case, _seed(name)))
    _run(d, case)  # first-call setup out of the trace
    torch.cuda.synchronize()
    spec = speculative(case, sms)
    want = _want_kernels(steps(case, sms))
    host_chfsi = not spec and any(p["eig"].startswith("chfsi") for p in steps(case, sms))
    solvers = {"jacobi2_f32", "jacobi2_f64", "jacobi2_mixed", "jacobi_f64", "cheb_filter", "chfsi", "chfsi_adaptive"}
    if host_chfsi:  # the host ChFSI's Rayleigh-Ritz solves and filter are not part of the restatement
        want -= solvers
    seen = set()
    # the activity trace occasionally comes back empty or missing records: take it again (never accept an empty one);
    # a path that differs from the restatement differs in every trace
    for _ in range(5):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            _, info = _run(d, case)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        seen = {what for n in names for key, what in _KERNELS.items() if key in n}
        if host_chfsi:
            seen -= solvers
        if names and seen == want:
            break
    assert names, "the profiler recorded no kernel"
    assert info["speculative"] == int(spec), (name, info)
    print(f"{name}: sms {sms}, launched {sorted(seen)}")
    assert seen == want, (name, sorted(seen), sorted(want))


# ==================================================================================================== batch
@pytest.mark.gpu
def test_batch_matches_single_calls():
    """ttsvd_batch with inflight = 8 on low-noise (rejected: bit 0) and randn (accepted) tensors interleaved: each
    tensor's cores and ranks match its single call, and its `speculative` entry the restatement."""
    from tntorch_b200 import ops

    low = CASES["lownoise_f32"]
    shape, r = low["shape"], low["rmax"]
    xs, want = [], []
    for i in range(10):
        c = dict(low) if i % 2 == 0 else dict(low, kind="randn", reject=False)
        xs.append(torch.as_tensor(make_input(c, 900 + i)).to(F32).cuda())
        want.append(0 if c.get("reject") else 1)
    got, info = ops.ttsvd_batch(xs, rmax=r, inflight=8, return_info=True)
    assert info["speculative"] == want, (info["speculative"], want)
    worst = 0.0
    for x, cores in zip(xs, got):
        single = ops.ttsvd(x, rmax=r)
        assert ranks_of(cores) == ranks_of(single)
        X64 = x.double().cpu().numpy()
        worst = max(worst, abs(relerr(X64, host(cores)) - relerr(X64, host(single))))
    print(f"batch: speculative {info['speculative']}, largest relerr difference to the single calls {worst:.1e}")
    assert worst <= TOL[F32]["relerr"], worst
