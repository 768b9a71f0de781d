"""CPU: tnb_tt_dot is sized without a GPU and its size is restated from the shapes (one F per pair and one mode's
partial sums, never a copy of a core), unsupported dtypes size to 0 and are refused with TNB_ERR_UNSUPPORTED, malformed
arguments get their codes before anything is launched, no host synchronisation is on the path (checked on the source),
and the CPU restatement of the chooser is the source's."""
import ctypes
import os
import re

import ttd_model as tm
from tntorch_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64 = _lib.TNB_F32, _lib.TNB_F64

# (shape, per-pair ranks of a, per-pair ranks of b)
CASES = [
    ([7], [[1, 1]], [[1, 1]]),
    ([128] * 10, [[1] + [64] * 9 + [1]], [[1] + [16] * 9 + [1]]),
    ([128] * 10, [[1] + [64] * 9 + [1]] * 64, [[1] + [64] * 9 + [1]] * 64),
    ([64] * 8, [[1, 64, 256, 256, 256, 256, 256, 64, 1]], [[1, 64, 256, 256, 256, 256, 256, 64, 1]]),
    ([3, 1, 5, 1, 2], [[1, 3, 3, 5, 2, 1], [1, 2, 2, 2, 2, 1]], [[1, 1, 1, 4, 2, 1], [1, 3, 3, 7, 2, 1]]),
    ([40, 50, 60], [[1, 40, 300, 1]], [[1, 20, 17, 1]]),
    ([9] * 4, [[1, 9, 81, 9, 1]] * 70, [[1, 9, 20, 9, 1]] * 70),
]


def _flat(rs):
    return [x for r in rs for x in r]


def _size(dtype, shape, ra, rb, npairs=None):
    P = len(ra) if npairs is None else npairs
    return _lib.lib().tnb_tt_dot_workspace_bytes(dtype, P, len(shape), _lib.i64(shape), _lib.i32(_flat(ra)),
                                                 _lib.i32(_flat(rb)))


def _call(dtype, shape, ra, rb, npairs=None, a=1, b=1, out=1, ws=1, ws_bytes=1 << 40, nulls=()):
    """The run entry with dummy non-null pointers: every check below fails before anything is dereferenced."""
    P = len(ra) if npairs is None else npairs
    n = max(P * len(shape), 1)
    buf = (ctypes.c_double * 8)()
    p = ctypes.c_void_p(ctypes.addressof(buf))
    ptrs = (ctypes.c_void_p * n)(*([ctypes.addressof(buf)] * n))
    return _lib.lib().tnb_tt_dot(dtype, ptrs if a else None, ptrs if b else None, P, len(shape),
                                 None if "s" in nulls else _lib.i64(shape), None if "a" in nulls else _lib.i32(_flat(ra)),
                                 None if "b" in nulls else _lib.i32(_flat(rb)), p if out else None, p if ws else None,
                                 ws_bytes, None)


def test_workspace_is_restated_from_the_shapes():
    for shape, ra, rb in CASES:
        for dt in (F32, F64):
            assert _size(dt, shape, ra, rb) == tm.workspace_bytes(shape, ra, rb), (shape, dt)


def test_workspace_never_holds_a_core():
    """Config 3 (128^10, rank 64): a core is 4 MB; the workspace is one 64 x 64 F and the partials of 128 chunks."""
    shape, ra, rb = CASES[2][0], CASES[2][1][:1], CASES[2][2][:1]
    assert _size(F64, shape, ra, rb) == 64 * 64 * 8 + 128 * 64 * 64 * 8
    # a batch of 64: 64 F blocks, 4 chunks per pair
    shape, ra, rb = CASES[2]
    assert _size(F64, shape, ra, rb) == 64 * 64 * 64 * 8 + 64 * 4 * 64 * 64 * 8


def test_supported_calls_never_size_to_zero():
    for dt in (F32, F64):
        assert _size(dt, [1], [[1, 1]], [[1, 1]]) >= 256


def test_unsupported_dtypes_size_to_zero_and_are_refused():
    for dt in (_lib.TNB_BF16, _lib.TNB_F16, _lib.TNB_F8E4M3, _lib.TNB_F8E5M2, 7, -1):
        assert _size(dt, [8, 8], [[1, 4, 1]], [[1, 4, 1]]) == 0
        assert _call(dt, [8, 8], [[1, 4, 1]], [[1, 4, 1]]) == _lib.ERR_UNSUPPORTED
        assert b"not built" in _lib.lib().tnb_last_error()


def test_malformed_arguments_get_their_codes():
    shape, ra, rb = [4, 5, 6], [[1, 3, 3, 1]], [[1, 2, 2, 1]]
    invalid = [(shape, [[2, 3, 3, 1]], rb, None), (shape, ra, [[1, 2, 2, 3]], None),   # boundary ranks
               ([4, 0, 6], ra, rb, None), (shape, [[1, 0, 3, 1]], rb, None),          # sizes and ranks below 1
               ([], [[1]], [[1]], None),                                              # ndim < 1
               (shape, ra, rb, 0), (shape, ra, rb, -2)]                               # npairs < 1
    for s, a, b, P in invalid:
        assert _size(F32, s, a, b, P) == 0, (s, a, b, P)
        assert _call(F32, s, a, b, P) == _lib.ERR_INVALID, (s, a, b, P)
    for kw in (dict(a=0), dict(b=0), dict(out=0), dict(ws=0), dict(nulls="s"), dict(nulls="a"), dict(nulls="b")):
        assert _call(F64, shape, ra, rb, **kw) == _lib.ERR_INVALID, kw
    L = _lib.lib()
    assert L.tnb_tt_dot_workspace_bytes(F32, 1, 3, None, _lib.i32(ra[0]), _lib.i32(rb[0])) == 0
    assert L.tnb_tt_dot_workspace_bytes(F32, 1, 3, _lib.i64(shape), _lib.i32(ra[0]), None) == 0
    # too large: refused, not mis-sized
    for s, a in (([1 << 47], [[1, 1]]), ([2, 2], [[1, 1 << 26, 1]]), ([2] * 1025, [[1] * 1026])):
        assert _size(F32, s, a, a) == 0
        assert _call(F32, s, a, a) == _lib.ERR_UNSUPPORTED


def test_small_workspace_is_refused_before_any_launch():
    """A workspace below the size is TNB_ERR_WORKSPACE (or, here without a device, the device error that precedes it),
    never a launch."""
    shape, ra, rb = [4, 5, 6], [[1, 3, 3, 1]], [[1, 2, 2, 1]]
    before = _lib.lib().tnb_launch_count()
    assert _call(F64, shape, ra, rb, ws_bytes=16) in (_lib.ERR_WORKSPACE, _lib.ERR_CUDA)
    assert _lib.lib().tnb_launch_count() == before


def test_no_host_synchronisation_on_the_path():
    csrc = os.path.join(REPO, "tntorch_b200", "csrc")
    banned = re.compile(r"cuda(Stream|Device|Event)Synchronize|cudaMemcpy|cudaMalloc|cudaFree|pinned_scratch|\batomic[A-Z]")
    assert not banned.search(open(os.path.join(csrc, "tt_dot.cuh")).read())
    src = open(os.path.join(csrc, "tnb200.cu")).read()
    body = src[src.index("int tnb_tt_dot("):]
    body = body[: body.index("\n}\n")]
    assert "tt_dot_impl" in body and not banned.search(body)
    ops = open(os.path.join(REPO, "tntorch_b200", "ops.py")).read()
    fn = ops[ops.index("def tt_dot_batch("):]
    assert not re.search(r"\.item\(|\.cpu\(|\.tolist\(|synchronize|\.numpy\(|float\(", fn)


def test_chooser_restatement_matches_the_source():
    """The constants and formulas of the CPU restatement are the header's."""
    src = open(os.path.join(REPO, "tntorch_b200", "csrc", "tt_dot.cuh")).read()
    for c in ("TTD_TC_MAX_R = 256;", "TTD_TC_MIN_R = 16;", "TTD_BM = 32;", "TTD_GN = 64;", "TTD_TARGET_ITEMS = 512;",
              "TTD_GROUP = 32;"):
        assert c in src, c
    assert "return rbo * ra * (rb + rao) < rao * rb * (ra + rbo);" in src
    assert tm.order(64, 16, 16, 64) is False and tm.order(16, 64, 64, 16) is True and tm.order(64, 64, 64, 64) is False
    assert tm.mode_path(64, 64, 64, 64) == tm.TC and tm.mode_path(1, 1, 64, 64) == tm.RANK_MIN
    assert tm.mode_path(300, 20, 20, 20) == tm.RANK_MAX


def test_every_chooser_path_has_a_gpu_case():
    """tests/test_gpu_tt_dot.py names a case for every branch of ttd_mode_path."""
    import test_gpu_tt_dot as g

    seen = set()
    for shape, ra, rb in g.PATH_CASES.values():
        for row in tm.paths(shape, [[1] + ra + [1]], [[1] + rb + [1]]):
            seen.update(row)
    assert seen == set(tm.BRANCHES), seen
    assert set(g.PATH_CASES) >= {tm.BRANCHES[b] for b in tm.BRANCHES}
