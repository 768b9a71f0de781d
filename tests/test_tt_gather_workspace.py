"""CPU: tnb_tt_gather is sized without a GPU and its size is restated from the shapes (the narrowed indices, one
permutation and tile list, two state buffers; never a copy of a core, and nothing on the fused path), unsupported dtypes
size to 0 and are refused, malformed arguments get their codes before anything is launched, and every branch of both
choosers is reached by a case of tests/test_gpu_tt_gather.py."""
import ctypes
import os
import re

import ttg_model as tm
from tntorch_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64 = _lib.TNB_F32, _lib.TNB_F64

# (shape, per-train ranks, first, last, P)
CASES = [
    ([7], [[1, 1]], 0, 1, 1),
    ([32] * 6, [[1] + [10] * 5 + [1]], 0, 6, 1000),
    ([128] * 10, [[1] + [64] * 9 + [1]], 0, 10, 1 << 20),
    ([64] * 5, [[1] + [32] * 4 + [1]], 0, 5, 1 << 22),
    ([16] * 8, [[1, 16, 256, 256, 256, 256, 256, 16, 1]], 0, 8, 1 << 16),
    ([4, 5, 6, 3], [[1, 3, 4, 2, 1], [1, 2, 5, 2, 1]], 1, 3, 7),
    ([9, 1, 300], [[1, 9, 9, 1]] * 3, 0, 3, 5000),
    ([8] * 70, [[1] + [2] * 69 + [1]], 0, 70, 3),
]


def _flat(rs):
    return [x for r in rs for x in r]


def _size(dtype, shape, ranks, first, last, P, ntrains=None):
    nt = len(ranks) if ntrains is None else ntrains
    return _lib.lib().tnb_tt_gather_workspace_bytes(dtype, nt, len(shape), _lib.i64(shape), _lib.i32(_flat(ranks)),
                                                    first, last, P)


def _call(dtype, shape, ranks, first, last, P, ntrains=None, cores=1, idx=1, out=1, ws=1, ws_bytes=1 << 40, nulls=()):
    """The run entry with dummy non-null pointers: every check below fails before anything is dereferenced."""
    nt = len(ranks) if ntrains is None else ntrains
    n = max(nt * len(shape), 1)
    buf = (ctypes.c_double * 8)()
    p = ctypes.c_void_p(ctypes.addressof(buf))
    ptrs = (ctypes.c_void_p * n)(*([ctypes.addressof(buf)] * n))
    return _lib.lib().tnb_tt_gather(dtype, ptrs if cores else None, nt, len(shape),
                                    None if "s" in nulls else _lib.i64(shape),
                                    None if "r" in nulls else _lib.i32(_flat(ranks)), first, last, p if idx else None, P,
                                    p if out else None, p if ws else None, ws_bytes, None)


def test_workspace_is_restated_from_the_shapes():
    for shape, ranks, first, last, P in CASES:
        for dt, es in ((F32, 4), (F64, 8)):
            assert _size(dt, shape, ranks, first, last, P) == tm.workspace_bytes(shape, ranks, first, last, P, es), \
                (shape, dt)


def test_workspace_never_holds_a_core():
    """Config 3 at P = 2^20: indices, counts, tiles, one permutation and two states of P x 64; a core is 8 MB."""
    shape, ranks, first, last, P = CASES[2]
    ws = _size(F64, shape, ranks, first, last, P)
    assert 2 * P * 64 * 8 < ws <= 2 * P * 64 * 8 + P * 10 * 4 + P * 4 + 3 * 4 * (P // 64 + 129) + 4096
    assert _size(F64, *CASES[1]) == 256  # fused: nothing


def test_unsupported_dtypes_size_to_zero_and_are_refused():
    for dt in (_lib.TNB_BF16, _lib.TNB_F16, _lib.TNB_F8E4M3, _lib.TNB_F8E5M2, 7, -1):
        assert _size(dt, [8, 8], [[1, 4, 1]], 0, 2, 3) == 0
        assert _call(dt, [8, 8], [[1, 4, 1]], 0, 2, 3) == _lib.ERR_UNSUPPORTED
        assert b"not built" in _lib.lib().tnb_last_error()


def test_malformed_arguments_get_their_codes():
    shape, ranks = [4, 5, 6], [[1, 3, 3, 1]]
    invalid = [(shape, ranks, 1, 1, 3, None), (shape, ranks, 2, 1, 3, None), (shape, ranks, -1, 2, 3, None),
               (shape, ranks, 0, 4, 3, None),                                              # the range
               ([4, 0, 6], ranks, 0, 3, 3, None), (shape, [[1, 0, 3, 1]], 0, 3, 3, None),  # sizes and ranks below 1
               (shape, ranks, 0, 3, 0, None), (shape, ranks, 0, 3, -5, None),              # npoints < 1
               (shape, ranks, 0, 3, 3, 0)]                                                 # ntrains < 1
    for s, r, f, l, P, nt in invalid:
        assert _size(F32, s, r, f, l, P, nt) == 0, (s, r, f, l, P, nt)
        assert _call(F32, s, r, f, l, P, nt) == _lib.ERR_INVALID, (s, r, f, l, P, nt)
    for kw in (dict(cores=0), dict(idx=0), dict(out=0), dict(ws=0), dict(nulls="s"), dict(nulls="r")):
        assert _call(F64, shape, ranks, 0, 3, 3, **kw) == _lib.ERR_INVALID, kw
    # too large: refused, not mis-sized
    for s, r, P in (([1 << 47], [[1, 1]], 1), ([2, 2], [[1, 1 << 21, 1]], 1), ([2] * 1025, [[1] * 1026], 1),
                    ([1 << 31], [[1, 1]], 1), ([4, 4], [[64, 4, 1]], 1 << 25),
                    ([4, 4], [[1, 1 << 20, 1]], 1 << 27)):
        assert _size(F32, s, r, 0, len(s), P) == 0, (s, P)
        assert _call(F32, s, r, 0, len(s), P) == _lib.ERR_UNSUPPORTED, (s, P)


def test_small_workspace_is_refused_before_any_launch():
    shape, ranks = [4, 5, 6], [[1, 3, 3, 1]]
    before = _lib.lib().tnb_launch_count()
    assert _call(F64, shape, ranks, 0, 3, 5000, ws_bytes=16) in (_lib.ERR_WORKSPACE, _lib.ERR_CUDA)
    assert _lib.lib().tnb_launch_count() == before


def test_no_host_synchronisation_on_the_path():
    csrc = os.path.join(REPO, "tntorch_b200", "csrc")
    banned = re.compile(r"cuda(Stream|Device|Event)Synchronize|cudaMemcpy|cudaMalloc|cudaFree|pinned_scratch")
    assert not banned.search(open(os.path.join(csrc, "tt_gather.cuh")).read())
    src = open(os.path.join(csrc, "tnb200.cu")).read()
    body = src[src.index("int tnb_tt_gather("):]
    body = body[: body.index("\n}\n")]
    assert "tt_gather_impl" in body and not banned.search(body)


def test_chooser_restatement_matches_the_source():
    src = open(os.path.join(REPO, "tntorch_b200", "csrc", "tt_gather.cuh")).read()
    for c in ("TTG_TC_MIN_R = 16;", "TTG_TC_MAX_R = 256;", "TTG_FUSED_MAX_ROWS = 4096;", "TTG_FUSED_MAX_STATE = 2048;",
              "TTG_FUSED_MAX_MODES = 64;", "TTG_T = 64;"):
        assert c in src, c
    assert tm.path([[1, 10, 10, 1]], 0, 3, 1000) == tm.FUSED and tm.path([[1, 10, 10, 1]], 0, 3, 5000) == tm.GROUPED
    assert tm.path([[1, 64, 64, 1]], 0, 3, 10) == tm.FUSED and tm.path([[1, 4096, 4, 1]], 0, 3, 1) == tm.GROUPED
    assert tm.path([[1] * 66], 0, 65, 1) == tm.GROUPED
    assert tm.mode_path(16, 256) == tm.TC and tm.mode_path(15, 64) == tm.RANK_MIN and tm.mode_path(16, 257) == tm.RANK_MAX


def test_every_chooser_branch_has_a_gpu_case():
    """tests/test_gpu_tt_gather.py names a case for every branch of ttg_path and of ttg_mode_path."""
    import test_gpu_tt_gather as g

    paths, modes = set(), set()
    for shape, r, first, last, P in g.PATH_CASES.values():
        paths.add(tm.path([r], first, last, P))
        if tm.path([r], first, last, P) == tm.GROUPED:
            modes.update(tm.mode_paths(r, first, last))
    assert paths == set(tm.PATHS) and modes == set(tm.BRANCHES), (paths, modes)
