"""CPU: tnb_tt_gather_grad is sized without a GPU and its size is restated from the shapes (tests/ttgg_model.py: the
narrowed indices, per-mode counts and stable orders, the sort buffers, one train's tile and chunk lists, the kept L_k,
two W buffers and one mode's chunk partials; never a copy of a core), unsupported dtypes size to 0 and are refused, and
malformed arguments get their codes before anything is dereferenced or launched."""
import ctypes
import os
import re

import ttgg_model as gm
from tntorch_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64 = _lib.TNB_F32, _lib.TNB_F64

# (shape, per-train ranks, first, last, P)
CASES = [
    ([7], [[1, 1]], 0, 1, 1),
    ([32] * 6, [[1] + [10] * 5 + [1]], 0, 6, 1 << 16),
    ([128] * 10, [[1] + [64] * 9 + [1]], 0, 10, 1 << 20),
    ([64] * 5, [[1] + [32] * 4 + [1]], 0, 5, 1 << 22),
    ([2] * 20, [[1] + [16] * 19 + [1]], 0, 20, 1 << 18),
    ([4, 5, 6, 3], [[1, 3, 4, 2, 1], [1, 2, 5, 2, 1]], 1, 3, 7),
    ([9, 1, 300], [[1, 9, 9, 1]] * 3, 0, 3, 5000),
    ([600, 3], [[1, 20, 1]], 0, 2, 70000),
]


def _flat(rs):
    return [x for r in rs for x in r]


def _size(dtype, shape, ranks, first, last, P, ntrains=None):
    nt = len(ranks) if ntrains is None else ntrains
    return _lib.lib().tnb_tt_gather_grad_workspace_bytes(dtype, nt, len(shape), _lib.i64(shape),
                                                         _lib.i32(_flat(ranks)), first, last, P)


def _call(dtype, shape, ranks, first, last, P, ntrains=None, cores=1, idx=1, gout=1, grads=1, ws=1, ws_bytes=1 << 40,
          nulls=()):
    """The run entry with dummy non-null pointers: every check below fails before anything is dereferenced."""
    nt = len(ranks) if ntrains is None else ntrains
    n = max(nt * len(shape), 1)
    buf = (ctypes.c_double * 8)()
    p = ctypes.c_void_p(ctypes.addressof(buf))
    ptrs = (ctypes.c_void_p * n)(*([ctypes.addressof(buf)] * n))
    gptrs = (ctypes.c_void_p * n)(*([None if "g" in nulls else ctypes.addressof(buf)] * n))
    return _lib.lib().tnb_tt_gather_grad(dtype, ptrs if cores else None, nt, len(shape),
                                         None if "s" in nulls else _lib.i64(shape),
                                         None if "r" in nulls else _lib.i32(_flat(ranks)), first, last,
                                         p if idx else None, P, p if gout else None, gptrs if grads else None,
                                         p if ws else None, ws_bytes, None)


def test_workspace_is_restated_from_the_shapes():
    for shape, ranks, first, last, P in CASES:
        for dt, es in ((F32, 4), (F64, 8)):
            assert _size(dt, shape, ranks, first, last, P) == gm.workspace_bytes(shape, ranks, first, last, P, es), \
                (shape, dt)


def test_workspace_never_holds_a_core():
    """Config 3 at P = 2^20: the kept L_k (P x 64 x 9), two W buffers, orders, lists and partials; a core is 8 MB and
    the workspace is within a few percent of the states alone."""
    shape, ranks, first, last, P = CASES[2]
    ws = _size(F64, shape, ranks, first, last, P)
    states = P * 64 * 9 * 8 + 2 * P * 64 * 8
    assert states < ws < states * 1.1


def test_unsupported_dtypes_size_to_zero_and_are_refused():
    for dt in (_lib.TNB_BF16, _lib.TNB_F16, _lib.TNB_F8E4M3, _lib.TNB_F8E5M2, 7, -1):
        assert _size(dt, [8, 8], [[1, 4, 1]], 0, 2, 3) == 0
        assert _call(dt, [8, 8], [[1, 4, 1]], 0, 2, 3) == _lib.ERR_UNSUPPORTED
        assert b"not built" in _lib.lib().tnb_last_error()


def test_malformed_arguments_get_their_codes():
    shape, ranks = [4, 5, 6], [[1, 3, 3, 1]]
    invalid = [(shape, ranks, 1, 1, 3, None), (shape, ranks, 2, 1, 3, None), (shape, ranks, -1, 2, 3, None),
               (shape, ranks, 0, 4, 3, None),
               ([4, 0, 6], ranks, 0, 3, 3, None), (shape, [[1, 0, 3, 1]], 0, 3, 3, None),
               (shape, ranks, 0, 3, 0, None), (shape, ranks, 0, 3, -5, None),
               (shape, ranks, 0, 3, 3, 0)]
    for s, r, f, l, P, nt in invalid:
        assert _size(F32, s, r, f, l, P, nt) == 0, (s, r, f, l, P, nt)
        assert _call(F32, s, r, f, l, P, nt) == _lib.ERR_INVALID, (s, r, f, l, P, nt)
    for kw in (dict(cores=0), dict(idx=0), dict(gout=0), dict(grads=0), dict(ws=0), dict(nulls="s"),
               dict(nulls="r"), dict(nulls="g")):
        assert _call(F64, shape, ranks, 0, 3, 3, **kw) == _lib.ERR_INVALID, kw
    for s, r, P in (([1 << 47], [[1, 1]], 1), ([2, 2], [[1, 1 << 21, 1]], 1), ([2] * 1025, [[1] * 1026], 1),
                    ([1 << 31], [[1, 1]], 1), ([4, 4], [[64, 4, 1]], 1 << 25)):
        assert _size(F32, s, r, 0, len(s), P) == 0, (s, P)
        assert _call(F32, s, r, 0, len(s), P) == _lib.ERR_UNSUPPORTED, (s, P)


def test_small_workspace_is_refused_before_any_launch():
    shape, ranks = [4, 5, 6], [[1, 3, 3, 1]]
    before = _lib.lib().tnb_launch_count()
    assert _call(F64, shape, ranks, 0, 3, 5000, ws_bytes=16) in (_lib.ERR_WORKSPACE, _lib.ERR_CUDA)
    assert _lib.lib().tnb_launch_count() == before


def test_no_host_synchronisation_on_the_path():
    csrc = os.path.join(REPO, "tntorch_b200", "csrc")
    banned = re.compile(r"cuda(Stream|Device|Event)Synchronize|cudaMemcpy|cudaMalloc|cudaFree|pinned_scratch|atomicAdd\(\s*s\.")
    assert not banned.search(open(os.path.join(csrc, "tt_gather_grad.cuh")).read())
    src = open(os.path.join(csrc, "tnb200.cu")).read()
    body = src[src.index("int tnb_tt_gather_grad("):]
    body = body[: body.index("\n}\n")]
    assert "tt_gather_grad_impl" in body and not banned.search(body)


def test_chooser_restatement_matches_the_source():
    src = open(os.path.join(REPO, "tntorch_b200", "csrc", "tt_gather_grad.cuh")).read()
    for c in ("TTGG_SORT_THREADS = 256;", "TTGG_SORT_ITEMS = 16;", "TTGG_CHUNK_MIN = 256;", "TTGG_CHUNK_MAX = 1 << 16;",
              "TTGG_CHUNK_CTAS = 1024;"):
        assert c in src, c
    assert gm.sort_passes(255) == 1 and gm.sort_passes(256) == 2 and gm.sort_passes(1 << 16) == 3
    assert gm.chunk_rows(1 << 20, 64, 64) == 1024 and gm.chunk_rows(1 << 18, 16, 16) == 256
    assert gm.chunk_rows(1 << 30, 1, 1) == 1 << 16
