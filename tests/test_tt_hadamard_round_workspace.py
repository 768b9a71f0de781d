"""CPU: tnb_tt_hadamard_round is sized without a GPU, its capacity and offsets are restated from the shapes
(tests/tthr_model.py), its workspace holds every left Gram and never the Kronecker cores, malformed arguments are refused
with their codes before anything is launched, the eigen envelope is refused at sizing, and the CPU restatement of the
path choosers covers every branch of the source's."""
import ctypes
import os
import re

import pytest

import tthr_model as hm
from tntorch_b200 import _lib, ops

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64 = _lib.TNB_F32, _lib.TNB_F64
SRC = os.path.join(REPO, "tntorch_b200", "csrc", "tt_hadamard_round.cuh")

CASES = [
    # shape, ranks a, ranks b, rmax
    ([9], [1, 1], [1, 1], None),
    ([7, 9], [1, 5, 1], [1, 4, 1], None),
    ([8] * 6, [1] + [24] * 5 + [1], [1] + [24] * 5 + [1], [20] * 5),
    ([128] * 10, [1] + [64] * 9 + [1], [1] + [64] * 9 + [1], [16] * 9),
    ([64] * 5, [1] + [32] * 4 + [1], [1] + [32] * 4 + [1], [32] * 4),
    ([32] * 8, [1] + [16] * 7 + [1], [1] + [16] * 7 + [1], None),
]


def _rm(rmax, N):
    return _lib.i32(rmax if rmax is not None else [0] * max(N - 1, 1))


def _cap(shape, ra, rb, rmax):
    N = len(shape)
    offs = (ctypes.c_int64 * N)()
    cap = _lib.lib().tnb_tt_hadamard_round_cores_capacity(N, _lib.i64(shape), _lib.i32(ra), _lib.i32(rb), _rm(rmax, N), offs)
    return cap, list(offs)


def _ws(dtype, shape, ra, rb, rmax):
    N = len(shape)
    return _lib.lib().tnb_tt_hadamard_round_workspace_bytes(dtype, N, _lib.i64(shape), _lib.i32(ra), _lib.i32(rb), _rm(rmax, N))


@pytest.mark.parametrize("case", range(len(CASES)))
def test_capacity_and_offsets_restated(case):
    shape, ra, rb, rmax = CASES[case]
    cap, offs = _cap(shape, ra, rb, rmax)
    d = hm.dims(shape, ra, rb, rmax)
    assert cap == d["capacity"]
    assert offs == d["slot"]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_workspace_holds_the_grams_not_the_kronecker_cores(case):
    shape, ra, rb, rmax = CASES[case]
    N = len(shape)
    R = [a * b for a, b in zip(ra, rb)]
    for dt in (F32, F64):
        w = _ws(dt, shape, ra, rb, rmax)
        assert w > 0
        grams = sum(r * r for r in R[:N]) * 8
        assert w >= grams
        chunks = max([hm.chunk(shape[k], ra[k], rb[k], ra[k + 1], rb[k + 1]) *
                      (max(rb[k] * ra[k] * rb[k] * ra[k + 1], rb[k] * ra[k + 1] * rb[k + 1] * ra[k + 1]) +
                       ra[k] * rb[k] * ra[k + 1] * rb[k + 1]) for k in range(N - 1)] or [0]) * 8
        d = hm.dims(shape, ra, rb, rmax)
        bond = max([(3 * R[mu] * shape[mu] * d["rcap"][mu + 1] + 3 * (shape[mu] * d["rcap"][mu + 1]) ** 2) * 8
                    for mu in range(N)])
        # the grams, the larger of the recurrence's chunk buffers and one bond's scratch, plus the sizing slack
        assert w <= 2 * (grams + max(chunks, bond)) + (64 << 20)
        kron = sum(R[k] * shape[k] * R[k + 1] for k in range(N)) * 8
        if kron > (8 << 30):
            assert w < kron // 4


def test_config3_workspace_measured_from_shapes():
    shape, ra, rb, rmax = CASES[3]
    w = _ws(F64, shape, ra, rb, rmax)
    assert 1.0e9 < w < 2.5e9, w


def test_unsupported_dtype_and_envelope_size_to_zero():
    shape, ra, rb, rmax = CASES[1]
    assert _ws(_lib.TNB_BF16, shape, ra, rb, rmax) == 0
    # eps-only at config 3 squared: the bond Grams are wider than 256 and the kept rank is not capped: sized, the
    # subspace solver's adaptive k covers it; an rmax above 240 at such a bond is refused
    s, a, b, _ = CASES[3]
    assert _ws(F64, s, a, b, [250] * 9) == 0
    assert "subspace eigensolver" in _lib.lib().tnb_last_error().decode()


def _call(shape, ra, rb, rmax=None, dtype=F64, a=1, b=1, out=1, ws=1, ws_bytes=1 << 40, cap=1 << 40, nulls=()):
    N = len(shape)
    pa = (ctypes.c_void_p * N)(*([a] * N))
    pb = (ctypes.c_void_p * N)(*([b] * N))
    rk = (ctypes.c_int32 * (N + 1))()
    en = (ctypes.c_double * 2)()
    args = dict(pa=pa, pb=pb, shape=_lib.i64(shape), ra=_lib.i32(ra), rb=_lib.i32(rb), out=ctypes.c_void_p(out),
                ws=ctypes.c_void_p(ws), rk=rk)
    for k in nulls:
        args[k] = None
    return _lib.lib().tnb_tt_hadamard_round(dtype, args["pa"], args["pb"], N, args["shape"], args["ra"], args["rb"],
                                            _rm(rmax, N), 1e-10, 0, args["ws"], ws_bytes, args["out"], cap, args["rk"],
                                            en, None)


def test_refusals_before_launch():
    shape, ra, rb = [4, 5, 6], [1, 2, 3, 1], [1, 3, 2, 1]
    assert _call(shape, ra, rb, dtype=_lib.TNB_BF16) == _lib.ERR_UNSUPPORTED
    for k in ("pa", "pb", "shape", "ra", "rb", "out", "ws", "rk"):
        assert _call(shape, ra, rb, nulls=(k,)) == _lib.ERR_INVALID, k
    assert _call(shape, [2, 2, 3, 1], rb) == _lib.ERR_INVALID          # boundary rank
    assert _call(shape, ra, [1, 3, 2, 2]) == _lib.ERR_INVALID          # boundary rank
    assert _call([4, 0, 6], ra, rb) == _lib.ERR_INVALID                # mode size
    assert _call(shape, [1, 0, 3, 1], rb) == _lib.ERR_INVALID          # rank
    assert _call(shape, [1, 5000, 3, 1], rb) == _lib.ERR_UNSUPPORTED   # an operand rank above 4096
    assert _call(shape, [1, 300, 300, 1], [1, 300, 300, 1]) == _lib.ERR_UNSUPPORTED  # R above 65536
    assert _call(shape, ra, rb, cap=3) == _lib.ERR_WORKSPACE           # short cores buffer
    assert _call(shape, ra, rb, ws_bytes=64) == _lib.ERR_WORKSPACE     # short workspace


def test_no_host_synchronisation_in_the_recurrence():
    src = open(SRC).read()
    rec = src[src.index("// ---------------- left Grams"):src.index("// ---------------- truncation from the right")]
    assert "cudaStreamSynchronize" not in rec and "cudaMemcpy(" not in rec
    assert "atomic" not in src.replace("no atomics", "")


def _source_path(fn, *args):
    """The source's chooser, read from the header and evaluated on the CPU (the same thresholds as the model's)."""
    src = open(SRC).read()
    for name, val in re.findall(r"constexpr int (TTHR_TC_M(?:IN|AX)_R) = (\d+);", src):
        assert int(val) == {"TTHR_TC_MIN_R": hm.TC_MIN_R, "TTHR_TC_MAX_R": hm.TC_MAX_R}[name]
    return fn(*args)


@pytest.mark.parametrize("ranks,allow,want", [
    ((64, 64, 64, 64), True, hm.PATH_TC),
    ((16, 256, 16, 256), True, hm.PATH_TC),
    ((1, 1, 64, 64), True, hm.PATH_RANK_MIN),
    ((64, 15, 64, 64), True, hm.PATH_RANK_MIN),
    ((64, 257, 64, 64), True, hm.PATH_RANK_MAX),
    ((64, 64, 64, 64), False, hm.PATH_FORCED),
])
def test_mode_path_branches(ranks, allow, want):
    assert _source_path(hm.mode_path, *ranks, allow) == want


def test_bond_path_branches():
    assert hm.bond_path(2048, 4096) == hm.PATH_TC
    assert hm.bond_path(8, 4096) == hm.PATH_RANK_MIN
    assert hm.bond_path(2048, 1) == hm.PATH_RANK_MIN
    assert hm.bond_path(2048, 4096, False) == hm.PATH_FORCED


def test_chunk_restated():
    assert hm.chunk(128, 64, 64, 64, 64) == 2           # config 3 squared: two mode values per launch
    assert hm.chunk(32, 16, 16, 16, 16) == 32           # a whole mode in one launch
    assert hm.chunk(7, 1, 1, 5, 4) == 7


def test_routing_rule():
    # product rank above 256: always the fused call
    assert ops.hadamard_round_instead_of_kronecker([8] * 6, [1] + [24] * 5 + [1], [1] + [24] * 5 + [1], 8, 80 << 30)
    # product rank 256 that fits: today's path
    assert not ops.hadamard_round_instead_of_kronecker([32] * 8, [1] + [16] * 7 + [1], [1] + [16] * 7 + [1], 8, 80 << 30)
    # the same without the memory for the Kronecker cores: the fused call
    assert ops.hadamard_round_instead_of_kronecker([32] * 8, [1] + [16] * 7 + [1], [1] + [16] * 7 + [1], 8, 1 << 20)
