"""Seeded synthetic inputs shared by the golden-vector generator, the tests and bench.py.

Everything is drawn from ``numpy.random.default_rng(seed)`` (PCG64: bit-identical on
every machine), so the GPU box regenerates exactly the inputs the reference saw in
the build container.  Test infrastructure (see oracle/tt_oracle.py header).
"""
from __future__ import annotations

import numpy as np


def _rng(seed):
    return np.random.default_rng(seed)


def random_tt(shape, ranks, seed, dtype=np.float64):
    """Random TT cores [r_{k-1}, I_k, r_k] with N(0,1) entries (like tn.randn, create.py:210-357)."""
    rng = _rng(seed)
    N = len(shape)
    if not hasattr(ranks, "__len__"):
        ranks = [ranks] * (N - 1)
    rs = [1] + list(ranks) + [1]
    return [rng.standard_normal((rs[k], shape[k], rs[k + 1])).astype(dtype) for k in range(N)]


def tt_full(cores, dtype=None):
    f = np.ones((1, 1), dtype=cores[0].dtype)
    shape = []
    for c in cores:
        shape.append(c.shape[1])
        f = (f @ c.reshape(c.shape[0], -1)).reshape(-1, c.shape[2])
    out = f[:, 0].reshape(shape)
    return out if dtype is None else out.astype(dtype)


def analytic_field_128():
    """docs/tutorials/decompositions.ipynb:37 — the analytic 128^3 fp64 field."""
    X, Y, Z = np.meshgrid(range(128), range(128), range(128))
    return np.sqrt(np.sqrt(X) * (Y + Z) + Y * Z**2) * (X + np.sin(Y) * np.cos(Z))


def make_dense(spec):
    kind = spec["kind"]
    dtype = np.dtype(spec.get("dtype", "float32"))
    if kind == "randn":
        return _rng(spec["seed"]).standard_normal(spec["shape"]).astype(dtype)
    if kind == "tt_noise":  # structured twin: low TT-rank signal + relative Gaussian noise
        cores = random_tt(spec["shape"], spec["rank"], spec["seed"], np.float64)
        X = tt_full(cores)
        noise = _rng(spec["seed"] + 1).standard_normal(X.shape)
        X = X + spec["noise"] * X.std() * noise
        return X.astype(dtype)
    if kind == "analytic128":
        return analytic_field_128().astype(dtype)
    if kind == "smooth":  # fast-decaying singular spectrum
        grids = np.meshgrid(*[np.linspace(0, 1, s) for s in spec["shape"]], indexing="ij")
        X = 1.0 / (1.0 + sum((i + 1) * g for i, g in enumerate(grids)))
        return X.astype(dtype)
    if kind == "zeros":
        return np.zeros(spec["shape"], dtype)
    raise ValueError(kind)


def make_tt(spec):
    dtype = np.dtype(spec.get("dtype", "float64"))
    cores = random_tt(spec["shape"], spec["rank"], spec["seed"], dtype)
    if spec.get("doubled"):  # t + t : rank-doubling block cores (tensor.py:445-520 semantics)
        out = []
        N = len(cores)
        for k, c in enumerate(cores):
            r0, I, r1 = c.shape
            if k == 0:
                out.append(np.concatenate([c, c], axis=2))
            elif k == N - 1:
                out.append(np.concatenate([c, c], axis=0))
            else:
                z = np.zeros((2 * r0, I, 2 * r1), dtype)
                z[:r0, :, :r1] = c
                z[r0:, :, r1:] = c
                out.append(z)
        cores = out
    return cores


def make_matrix(spec):
    dtype = np.dtype(spec.get("dtype", "float64"))
    rng = _rng(spec["seed"])
    m, n = spec["shape"]
    if spec.get("lowrank"):
        k = spec["lowrank"]
        M = rng.standard_normal((m, k)) @ rng.standard_normal((k, n))
        M = M + spec.get("noise", 0.0) * rng.standard_normal((m, n))
    elif spec.get("zero"):
        M = np.zeros((m, n))
    else:
        M = rng.standard_normal((m, n))
    return M.astype(dtype)


def make_cp_dense(spec):
    rng = _rng(spec["seed"])
    dtype = np.dtype(spec.get("dtype", "float64"))
    fac = [rng.standard_normal((s, spec["Rtrue"])) for s in spec["shape"]]
    letters = "abcdefgh"[: len(fac)]
    X = np.einsum(",".join(f"{l}r" for l in letters) + "->" + letters, *fac)
    X = X + spec.get("noise", 0.0) * X.std() * rng.standard_normal(X.shape)
    return X.astype(dtype)


# ---- dense TT-SVD cases (tn.Tensor(X, ranks_tt=/eps=)) ------------------------------
TTSVD_CASES = {
    # BASELINE.json configs[0]
    "cfg1_randn16x4_f32": dict(kind="randn", shape=(16, 16, 16, 16), seed=0, dtype="float32", ranks_tt=4),
    "cfg1_randn16x4_f64": dict(kind="randn", shape=(16, 16, 16, 16), seed=0, dtype="float64", ranks_tt=4),
    # tests/test_gpu.py:9-27 precedent
    "gpu_randn16x3_r3": dict(kind="randn", shape=(16, 16, 16), seed=1, dtype="float32", ranks_tt=3),
    # ragged shapes, ranks list, rank larger than feasible
    "ragged_f32": dict(kind="randn", shape=(7, 12, 5, 9, 6), seed=2, dtype="float32", ranks_tt=[3, 8, 6, 2]),
    "ragged_f64_bigrank": dict(kind="randn", shape=(4, 6, 5, 3), seed=3, dtype="float64", ranks_tt=50),
    "two_modes": dict(kind="randn", shape=(40, 30), seed=4, dtype="float64", ranks_tt=5),
    # structured twins (meaningful error)
    "twin_small_f32": dict(kind="tt_noise", shape=(12, 10, 8, 9, 7), rank=4, noise=1e-2, seed=5, dtype="float32", ranks_tt=4),
    "twin_small_f64": dict(kind="tt_noise", shape=(12, 10, 8, 9, 7), rank=4, noise=1e-3, seed=5, dtype="float64", ranks_tt=4),
    "twin_16x5_f32": dict(kind="tt_noise", shape=(16,) * 5, rank=8, noise=1e-2, seed=6, dtype="float32", ranks_tt=8),
    # eps-driven
    "eps_twin_f64": dict(kind="tt_noise", shape=(12, 10, 8, 9, 7), rank=4, noise=1e-6, seed=7, dtype="float64", eps=1e-4),
    "eps_smooth_f64": dict(kind="smooth", shape=(20, 18, 16, 14), dtype="float64", eps=1e-6),
    "smooth_f32_r6": dict(kind="smooth", shape=(20, 18, 16, 14), dtype="float32", ranks_tt=6),
    # eps-only with a Gram matrix larger than the direct eigensolver (step 1: 320 / 288 columns): the leading values
    # come from the subspace iteration in growing blocks until the tail-energy rule is decided
    "eps_biggram_f32": dict(kind="tt_noise", shape=(40,) * 4, rank=8, noise=1e-3, seed=12, dtype="float32", eps=2e-2, big=True),
    # a finer budget (delta^2 / ||T||^2 = 1.3e-6): below the resolution of the TF32 Gram, the sweep must take the exact one
    "eps_fine_f32": dict(kind="tt_noise", shape=(40,) * 4, rank=8, noise=1e-4, seed=14, dtype="float32", eps=2e-3, big=True),
    "eps_biggram_f64": dict(kind="tt_noise", shape=(24,) * 4, rank=12, noise=1e-6, seed=13, dtype="float64", eps=1e-4),
    # tutorial known answers (docs/tutorials/decompositions.ipynb:68,361)
    "analytic128_r3": dict(kind="analytic128", dtype="float64", ranks_tt=3, big=False),
    "analytic128_eps": dict(kind="analytic128", dtype="float64", eps=1e-5, big=False),
    # medium: same character as BASELINE configs[1] (random Gaussian, r=32) at a CPU-feasible size
    "randn32x5_r32_f32": dict(kind="randn", shape=(32,) * 5, seed=8, dtype="float32", ranks_tt=32, big=True),
    "twin32x5_r32_f32": dict(kind="tt_noise", shape=(32,) * 5, rank=32, noise=1e-2, seed=9, dtype="float32", ranks_tt=32, big=True),
    "randn64x4_r32_f32": dict(kind="randn", shape=(64,) * 4, seed=10, dtype="float32", ranks_tt=32, big=True),
    "zeros": dict(kind="zeros", shape=(6, 5, 4), dtype="float64", ranks_tt=3),
}

# ---- round_tt on TT input ----------------------------------------------------------
ROUND_CASES = {
    "rmax_8to3_f64": dict(shape=(16,) * 5, rank=8, seed=20, dtype="float64", rmax=3),
    "rmax_list_f64": dict(shape=(9, 8, 7, 6, 5, 4), rank=6, seed=21, dtype="float64", rmax=[2, 4, 5, 3, 2]),
    "doubled_eps_f64": dict(shape=(8,) * 6, rank=5, seed=22, dtype="float64", doubled=True, eps=1e-8),
    "doubled_eps_f32": dict(shape=(8,) * 6, rank=5, seed=22, dtype="float32", doubled=True, eps=1e-4),
    "cfg3_small_f64": dict(shape=(32,) * 6, rank=16, seed=23, dtype="float64", rmax=4),
    "eps_only_f64": dict(shape=(10,) * 5, rank=7, seed=24, dtype="float64", eps=0.3),
}

# ---- truncated_svd ------------------------------------------------------------------
TSVD_CASES = {
    "rand_32x32_eps": dict(shape=(32, 32), seed=30, eps=0.3),
    "wide_16x200_rmax": dict(shape=(16, 200), seed=31, rmax=5),
    "tall_300x12_delta": dict(shape=(300, 12), seed=32, delta=2.0),
    "lowrank_60x80": dict(shape=(60, 80), seed=33, lowrank=6, noise=1e-9, eps=1e-6),
    "zero_10x7": dict(shape=(10, 7), seed=34, zero=True, rmax=3),
    "f32_64x128_rmax": dict(shape=(64, 128), seed=35, rmax=16, dtype="float32"),
    "lowrank_600x500_eps": dict(shape=(600, 500), seed=36, lowrank=20, noise=1e-6, eps=1e-4),
}

# ---- maxvol ---------------------------------------------------------------------------
MAXVOL_CASES = {
    "cfg5_320x10": dict(shape=(320, 10), seed=40),
    "tall_1000x20": dict(shape=(1000, 20), seed=41),
    "square_8x8": dict(shape=(8, 8), seed=42),
    "wide_5x7": dict(shape=(5, 7), seed=43),
    "small_64x8": dict(shape=(64, 8), seed=44),
}

# ---- CP-ALS (fp64 oracle, fixed sweep count: SURVEY §0.5) -------------------------------
CP_CASES = {
    "cp_16x4_R5": dict(shape=(16,) * 4, Rtrue=5, R=5, sweeps=10, noise=1e-2, seed=50, dtype="float64"),
    "cp_20x3_R8": dict(shape=(20, 18, 16), Rtrue=8, R=8, sweeps=8, noise=1e-3, seed=51, dtype="float64"),
    # five modes (every branch of the dimension-tree sweep: chain, inner modes, transposed last mode) and two modes
    "cp_5mode_R4": dict(shape=(8, 7, 6, 5, 9), Rtrue=4, R=4, sweeps=8, noise=1e-2, seed=52, dtype="float64"),
    "cp_2mode_R3": dict(shape=(30, 20), Rtrue=3, R=3, sweeps=4, noise=1e-2, seed=53, dtype="float64"),
}

# ---- TT-cross (seeded global NumPy/torch RNGs; function f(x) = 1 / (shift + sum_i x_i)) ----------------
CROSS_CASES = {
    "cfg5_32x6_r10": dict(N=6, I=32, lo=0.0, hi=1.0, shift=1.0, ranks_tt=10, max_iter=3, seed=60),
    "adaptive_32x5": dict(N=5, I=32, lo=1.0, hi=32.0, shift=0.0, kickrank=3, eps=1e-6, max_iter=25, seed=61),
    "small_10x3_r3": dict(N=3, I=10, lo=1.0, hi=10.0, shift=0.0, ranks_tt=3, max_iter=5, seed=62, forward=True),
    # _minimize mode (cross.py:342-359): sum_i (x_i - 0.37)^2 on a 16^4 grid, minimum 4 * 0.03^2 at index (6, 6, 6, 6)
    "minimize_16x4": dict(N=4, I=16, lo=0.0, hi=1.0, ranks_tt=4, max_iter=4, seed=63, minimize=True, fn="bowl"),
}


def cross_function(shift, fn=None):
    if fn == "bowl":
        def bowl(*xs):
            s = xs[0] * 0
            for x in xs:
                s = s + (x - 0.37) ** 2
            return s

        return bowl

    def f(*xs):
        s = xs[0] * 0 + shift
        for x in xs:
            s = s + x
        return 1.0 / s

    return f

# ---- Tucker rounding / tn.round / Tensor(eps=) (SURVEY §8f-2) ---------------------------------------------
TUCKER_CASES = {
    "dense_randn16x3_tucker3": dict(kind="dense", spec=dict(kind="randn", shape=(16, 16, 16), seed=70, dtype="float64"), ranks_tucker=3),
    "dense_analytic128_tucker3": dict(kind="dense", spec=dict(kind="analytic128", dtype="float64"), ranks_tucker=3),
    "dense_analytic128_eps": dict(kind="dense", spec=dict(kind="analytic128", dtype="float64"), eps=1e-5),
    "dense_twin_eps": dict(kind="dense", spec=dict(kind="tt_noise", shape=(12, 10, 8, 9, 7), rank=4, noise=1e-6, seed=7, dtype="float64"), eps=1e-4),
    "tt_round_tucker_eps": dict(kind="tt", spec=dict(shape=(16,) * 4, rank=6, seed=71, dtype="float64"), round_tucker=dict(eps=0.2)),
    "tt_round_tucker_rmax": dict(kind="tt", spec=dict(shape=(12, 14, 10, 9), rank=5, seed=72, dtype="float64"), round_tucker=dict(rmax=4)),
    "tt_round_eps": dict(kind="tt", spec=dict(shape=(10,) * 5, rank=7, seed=24, dtype="float64"), round=dict(eps=0.3)),
}
# further reference cases of the same layer (their goldens in tucker.npz too), whose inputs also take the "cp" kind and the
# Us / mode_rank / last_U_orthonormal fields of make_tucker_input; tests/test_gpu_tucker_paths.py runs every case of both
TUCKER_PATH_CASES = {
    # fp32 input, a capped rule on every mode
    "dense_twin_f32_tucker4": dict(kind="dense", spec=dict(kind="tt_noise", shape=(12, 10, 8, 9, 7), rank=4, noise=1e-2, seed=5, dtype="float32"), ranks_tucker=4),
    "dense_twin_f32_eps": dict(kind="dense", spec=dict(kind="tt_noise", shape=(12, 10, 8, 9, 7), rank=4, noise=1e-3, seed=7, dtype="float32"), eps=1e-2),
    # Tensor(X, ranks_tucker=, ranks_tt=): round_tucker, then round_tt
    "dense_twin_tucker_tt": dict(kind="dense", spec=dict(kind="tt_noise", shape=(12, 10, 8, 9, 7), rank=4, noise=1e-3, seed=73, dtype="float64"), ranks_tucker=5, ranks_tt=3),
    # rmax lists with None entries, rmax with eps, dim as a subset and as an int
    "tt_rmax_none_list": dict(kind="tt", spec=dict(shape=(12, 14, 10, 9), rank=5, seed=74, dtype="float64"), round_tucker=dict(rmax=[None, 3, None, 2])),
    "tt_eps_rmax": dict(kind="tt", spec=dict(shape=(16,) * 4, rank=6, seed=75, dtype="float64"), round_tucker=dict(eps=0.2, rmax=[16, 5, 16, 16])),
    "tt_dim_subset": dict(kind="tt", spec=dict(shape=(16,) * 4, rank=6, seed=76, dtype="float64"), round_tucker=dict(eps=0.2, dim=[0, 2])),
    "tt_dim_int": dict(kind="tt", spec=dict(shape=(16,) * 4, rank=6, seed=77, dtype="float64"), round_tucker=dict(eps=0.2, dim=1)),
    "tt_f32_eps": dict(kind="tt", spec=dict(shape=(16,) * 4, rank=6, seed=71, dtype="float32"), round_tucker=dict(eps=0.2)),
    # one and two modes
    "tt_N1": dict(kind="tt", spec=dict(shape=(30,), rank=1, seed=78, dtype="float64"), round_tucker=dict(eps=0.1)),
    "tt_N2": dict(kind="tt", spec=dict(shape=(40, 30), rank=6, seed=79, dtype="float64"), round_tucker=dict(rmax=4)),
    # TT-Tucker input (factors present, not orthonormal): rounded again
    "tucker_round_again": dict(kind="tt", spec=dict(shape=(5, 6, 4, 5), rank=3, seed=80, dtype="float64", Us=(12, 14, 10, 9)), round_tucker=dict(rmax=[4, 3, 4, 3])),
    # CP cores (first, middle and last) and CP cores under Tucker factors
    "cp_round_tucker": dict(kind="cp", spec=dict(shape=(10, 9, 8, 7), R=5, seed=81, dtype="float64"), round_tucker=dict(rmax=3)),
    "cp_tucker_round_tucker": dict(kind="cp", spec=dict(shape=(6, 5, 6), R=4, seed=82, dtype="float64", Us=(11, 12, 13)), round_tucker=dict(rmax=[4, 3, 4])),
    # the eigensolver ladder of the factor split, by L = min(I, k): mixed Jacobi (the 10s), two-sided fp64 (72), one-sided
    # in shared (100) and global memory (200), ChFSI (300 with rmax) and the adaptive solve (300, eps only, rank 30)
    "tt_L72": dict(kind="tt", spec=dict(shape=(9, 72, 9), rank=9, seed=83, dtype="float64", mode_rank={1: 12}), round_tucker=dict(eps=1e-6)),
    "tt_L100": dict(kind="tt", spec=dict(shape=(10, 100, 10), rank=10, seed=84, dtype="float64", mode_rank={1: 20}), round_tucker=dict(eps=1e-6)),
    "tt_L200": dict(kind="tt", spec=dict(shape=(15, 200, 15), rank=15, seed=85, dtype="float64", mode_rank={1: 25}), round_tucker=dict(eps=1e-6)),
    "tt_L300_chfsi": dict(kind="tt", spec=dict(shape=(18, 300, 18), rank=18, seed=86, dtype="float64", mode_rank={1: 30}), round_tucker=dict(rmax=[18, 20, 18])),
    "tt_L300_adaptive": dict(kind="tt", spec=dict(shape=(18, 300, 18), rank=18, seed=87, dtype="float64", mode_rank={1: 30}), round_tucker=dict(eps=1e-4)),
    # tn.round: the TT rounding reaches about 1e-8 (the dot formula's floor) of eps = 1e-4 on t + t and leaves the budget to round_tucker; with rmax = 2 it
    # reaches far more than eps and round_tucker is skipped
    "tt_round_leftover": dict(kind="tt", spec=dict(shape=(10, 11, 12, 13), rank=3, seed=88, dtype="float64", doubled=True), round=dict(eps=1e-4)),
    # tn.round on a TT-Tucker input whose factors 0..N-2 are not orthonormal: round_tt must push them into the cores first
    # (the reference pushes factors 0..N-2 only, tensor.py:2033, so the last one is drawn orthonormal)
    "tucker_round": dict(kind="tt", spec=dict(shape=(5, 6, 4, 5), rank=4, seed=90, dtype="float64", Us=(12, 14, 10, 9), last_U_orthonormal=True), round=dict(eps=0.3)),
    "tt_round_no_leftover": dict(kind="tt", spec=dict(shape=(10, 11, 12, 13), rank=6, seed=89, dtype="float64"), round=dict(eps=1e-3, rmax=2)),
}


def make_tucker_input(spec):
    """(cores, Us) of a TUCKER_CASES entry of kind "tt" or "cp".  "tt": random TT cores (make_tt), optionally with mode
    `mu`'s core projected onto a random `mode_rank[mu]`-dimensional subspace (its mode unfolding has that rank while
    r0 r1 and I stay large), optionally under random (not orthonormal) factors Us[n] [I_n, S_n].  "cp": random CP
    factors [S_n, R], optionally under factors.  Us is None where there is no factor."""
    dtype = np.dtype(spec.get("dtype", "float64"))
    rng = _rng(spec["seed"] + 1000)
    if "R" in spec:
        cores = [rng.standard_normal((S, spec["R"])).astype(dtype) for S in spec["shape"]]
    else:
        cores = make_tt(spec)
        for mu, k in spec.get("mode_rank", {}).items():
            c = cores[mu].astype(np.float64)
            P = np.linalg.qr(rng.standard_normal((c.shape[1], k)))[0]
            cores[mu] = np.einsum("aib,ij->ajb", c, P @ P.T).astype(dtype)
    Us = [None] * len(cores)
    if "Us" in spec:
        Us = [rng.standard_normal((I, c.shape[-2])).astype(dtype) for I, c in zip(spec["Us"], cores)]
        if spec.get("last_U_orthonormal"):
            Us[-1] = np.linalg.qr(Us[-1].astype(np.float64))[0].astype(dtype)
    return cores, Us


# ---- full-size cases of BASELINE.json configs 2-4 (golden outputs: oracle/gen_golden_full.py -> tests/golden/full.npz) -----
def make_dense_big(spec):
    """Full-size inputs, built in fp32 with bounded host memory (one 4 GiB array + one temporary)."""
    shape, seed = spec["shape"], spec["seed"]
    n = int(np.prod(shape))
    if spec["kind"] == "randn":
        return _rng(seed).standard_normal(n, dtype=np.float32).reshape(shape)
    if spec["kind"] == "tt_noise":
        cores = random_tt(shape, spec["rank"], seed, np.float64)
        h = len(shape) // 2
        left = tt_full_matrix(cores[:h]).astype(np.float32)          # (prod I_<h) x r
        right = tt_full_matrix(cores[h:], left_open=True).astype(np.float32)  # r x (prod I_>=h)
        X = left @ right
        std = float(np.sqrt(np.mean(np.square(X[:: max(1, X.shape[0] // 64)], dtype=np.float64))))
        noise = _rng(seed + 1).standard_normal(n, dtype=np.float32).reshape(X.shape)
        noise *= np.float32(spec["noise"] * std)
        X += noise
        return X.reshape(shape)
    raise ValueError(spec["kind"])


def tt_full_matrix(cores, left_open=False):
    """Contract a chain of TT cores into a matrix: (prod I) x r_last, or r_first x (prod I) when left_open."""
    if left_open:
        f = np.eye(cores[0].shape[0])
        for c in cores:
            f = (f.reshape(-1, c.shape[0]) @ c.reshape(c.shape[0], -1)).reshape(cores[0].shape[0], -1, c.shape[2])
            f = f.reshape(cores[0].shape[0], -1)
            f = f.reshape(cores[0].shape[0], -1, c.shape[2]).reshape(-1, c.shape[2]) if c is not cores[-1] else f
        return f.reshape(cores[0].shape[0], -1)
    f = np.ones((1, cores[0].shape[0]))
    for c in cores:
        f = (f @ c.reshape(c.shape[0], -1)).reshape(-1, c.shape[2])
    return f


FULL_TTSVD_CASES = {
    # BASELINE configs[1] stand-ins (SURVEY §8d): the bench tensor's character, and the structured twin
    "twin64x5_r32_f32": dict(kind="tt_noise", shape=(64,) * 5, rank=32, noise=1e-2, seed=109, dtype="float32", ranks_tt=32),
    "randn64x5_r32_f32": dict(kind="randn", shape=(64,) * 5, seed=108, dtype="float32", ranks_tt=32),
}
FULL_ROUND_CASES = {
    # BASELINE configs[2] exactly as named: tn.randn([128]*10, ranks_tt=64) -> round_tt(rmax=16), fp64
    "cfg3_128x10_r64to16_f64": dict(shape=(128,) * 10, rank=64, seed=123, dtype="float64", rmax=16),
    # reference tests/test_round.py:52-59 at that size: t + t -> round_tt(eps=1e-8) returns rank 64
    "cfg3_doubled_128x10_r32_f64": dict(shape=(128,) * 10, rank=32, seed=124, dtype="float64", doubled=True, eps=1e-8),
}
FULL_CP_CASES = {
    # BASELINE configs[3] at the CPU-feasible size of BASELINE.md §4: R=50 on 64^4, fp64 oracle, 10 sweeps
    "cp_64x4_R50": dict(shape=(64,) * 4, Rtrue=50, R=50, sweeps=10, noise=1e-2, seed=150, dtype="float64"),
}

# ---- fp32 inputs whose discarded tail is far below the TF32 noise floor of a tensor-core Gram (ADVICE r1): the sweep must
# ---- notice and take the exact Gram; rows >= 2048 at the first steps so that the tensor-core path is the default ----------
LOWNOISE_CASES = {
    "twin_lownoise_16x5_f32": dict(kind="tt_noise", shape=(16,) * 5, rank=6, noise=1e-5, seed=31, dtype="float32", ranks_tt=6),
    "smooth_24x4_f32_r5": dict(kind="smooth", shape=(24, 24, 24, 24), dtype="float32", ranks_tt=5),
}

# ---- rect_maxvol (maxvol.py:30-111): (matrix spec, keyword arguments) ----------------------------------------------------
RECT_MAXVOL_CASES = {
    "rect_320x10_tol1": (dict(shape=(320, 10), seed=40), dict(tol=1.0)),
    "rect_320x10_maxK15": (dict(shape=(320, 10), seed=40), dict(tol=0.5, maxK=15)),
    "rect_200x8_minK12": (dict(shape=(200, 8), seed=45), dict(tol=2.0, minK=12)),
    "rect_64x6_addK": (dict(shape=(64, 6), seed=46), dict(tol=1.0, min_add_K=3, maxK=20)),
    "rect_maxK_eq_r": (dict(shape=(320, 10), seed=40), dict(tol=1.0, maxK=10)),  # what tn.cross(_minimize=True) calls
}

# ---- batched TT-cross (BASELINE.json config 5): the family f_b(x) = 1 / (1 + b/512 + sum_i x_i) on [0, 1]^6, 32 points per
# ---- axis, ranks_tt = 10, 3 sweeps; golden = the first 16 problems run SEQUENTIALLY by the reference from one seed ------------
CROSS_BATCH_CASES = {
    # default eps = 1e-6: every problem converges after the first sweep and stops there (cross.py:461-462)
    "cfg5_default_eps": dict(N=6, I=32, lo=0.0, hi=1.0, ranks_tt=10, max_iter=3, seed=160, nproblems=16, family=512),
    # eps = 0: all three sweeps run
    "cfg5_three_sweeps": dict(N=6, I=32, lo=0.0, hi=1.0, ranks_tt=10, max_iter=3, eps=0.0, seed=161, nproblems=8, family=512),
}


def cross_family_function(b, family=512):
    def f(*xs):
        s = xs[0] * 0 + 1.0 + b / family
        for x in xs:
            s = s + x
        return 1.0 / s

    return f


# ---- callers that re-round in loops (SURVEY §8(f)-3): hadamard_sum, shift_mode, TTMatrix
HADAMARD_SUM_CASES = {
    "hs_3x_6545_r3": dict(shape=(6, 5, 4, 5), ranks=[(1, 3, 3, 3, 1), (1, 2, 4, 2, 1), (1, 3, 2, 3, 1)], seed=170),
    "hs_2x_8888_r5": dict(shape=(8, 8, 8, 8), ranks=[(1, 5, 5, 5, 1), (1, 4, 4, 4, 1)], seed=171),
    "hs_4x_444_r2": dict(shape=(4, 4, 4), ranks=[(1, 2, 2, 1)] * 4, seed=172),
}
SHIFT_MODE_CASES = {
    # (TT spec, mode, shift, eps)
    "shift_right2": (dict(shape=(4, 5, 6, 7), ranks=(1, 3, 4, 3, 1), seed=175), 0, 2, 1e-6),
    "shift_left3": (dict(shape=(4, 5, 6, 7), ranks=(1, 3, 4, 3, 1), seed=176), 3, -3, 1e-6),
    "shift_same": (dict(shape=(6, 6, 6, 6, 6), ranks=(1, 4, 4, 4, 4, 1), seed=177), 1, 2, "same"),
}
TTMATRIX_CASES = {
    # (matrix seed, input dims, output dims, ranks, batch)
    "ttm_16x24": dict(seed=180, input_dims=[4, 4], output_dims=[4, 6], ranks=[5], batch=0),
    "ttm_64x64_3": dict(seed=181, input_dims=[4, 4, 4], output_dims=[4, 4, 4], ranks=[6, 6], batch=0),
    "ttm_batch3_36x20": dict(seed=182, input_dims=[6, 6], output_dims=[4, 5], ranks=[7], batch=3),
}


def shift_mode_input(spec):
    return random_tt(spec["shape"], list(spec["ranks"][1:-1]), spec["seed"])


def hadamard_operands(spec):
    return [random_tt(spec["shape"], list(r[1:-1]), spec["seed"] + 13 * k) for k, r in enumerate(spec["ranks"])]


def ttmatrix_input(spec):
    import math

    rows, cols = math.prod(spec["input_dims"]), math.prod(spec["output_dims"])
    shape = ([spec["batch"]] if spec["batch"] else []) + [rows, cols]
    return _rng(spec["seed"]).standard_normal(shape)


def golden_prod(g, key):
    """L @ R of a truncated_svd.npz case: stored whole, or (to keep the file small) as the case's common column basis
    times per-key coefficients, exact to ~1e-15 relative."""
    if key + "/prod" in g.files:
        return g[key + "/prod"]
    return g[key.split("/")[0] + "/prod_basis"] @ g[key + "/prod_coef"]
