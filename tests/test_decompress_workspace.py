"""CPU: the TT -> dense entry point (tnb_tt_decompress) is sized without a GPU, its workspace cannot hold a dense image
of the result, every dtype pair it does not build sizes to 0 and is refused with TNB_ERR_UNSUPPORTED before any device
work, and bad arguments get their error codes.  No host synchronisation is on its path: the driver and the kernels
(csrc/expand_tc.cuh) contain no synchronising runtime call, which is checked on the source."""
import ctypes
import os
import re

from tntorch_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64, BF16, F16, E4, E5 = (_lib.TNB_F32, _lib.TNB_F64, _lib.TNB_BF16, _lib.TNB_F16, _lib.TNB_F8E4M3,
                               _lib.TNB_F8E5M2)
BUILT = [(F32, F32), (F32, BF16), (F32, F16), (F64, F64)]
REFUSED = [(F64, BF16), (F64, F16), (F64, F32), (F32, F64), (F32, E4), (F32, E5), (F64, E4), (BF16, BF16), (F16, F16),
           (BF16, F32), (F16, F32), (E4, F32), (7, F32), (F32, -1)]


def _size(core, out, shape, ranks):
    return _lib.lib().tnb_tt_decompress_workspace_bytes(core, out, len(shape), _lib.i64(shape), _lib.i32(ranks))


def _call(core, out, shape, ranks, cores=1, outp=1, ws=1, ws_bytes=1 << 20, shape_null=False, ranks_null=False):
    """The run entry with dummy non-null pointers: every check below fails before anything is dereferenced or launched."""
    N = len(shape)
    buf = (ctypes.c_double * 8)()
    ptrs = (ctypes.c_void_p * max(N, 1))(*([ctypes.addressof(buf)] * max(N, 1)))
    p = ctypes.c_void_p(ctypes.addressof(buf))
    return _lib.lib().tnb_tt_decompress(core, out, ptrs if cores else None, N, None if shape_null else _lib.i64(shape),
                                        None if ranks_null else _lib.i32(ranks), p if outp else None, p if ws else None,
                                        ws_bytes, None)


def test_flagship_workspace_cannot_hold_a_dense_image():
    shape, ranks = [64] * 5, [1, 32, 32, 32, 32, 1]
    for core, out in BUILT:
        ws = _size(core, out, shape, ranks)
        result_bytes = 64 ** 5 * {F32: 4, F64: 8, BF16: 2, F16: 2}[out]
        assert 0 < ws < result_bytes // 16, (core, out, ws)
    # the 16-bit outputs read the same fp32 operands: same workspace
    assert _size(F32, BF16, shape, ranks) == _size(F32, F16, shape, ranks) == _size(F32, F32, shape, ranks)


def test_supported_calls_never_size_to_zero():
    for shape, ranks in [([7], [1, 1]), ([3, 4], [1, 2, 1]), ([4, 5, 6], [1, 3, 3, 1]), ([2] * 40 + [1] * 22, [1] + [2] * 61 + [1])]:
        for core, out in BUILT:
            assert _size(core, out, shape, ranks) >= 256


def test_refused_pairs_size_to_zero_and_return_unsupported():
    shape, ranks = [4, 5, 6], [1, 3, 3, 1]
    for core, out in REFUSED:
        assert _size(core, out, shape, ranks) == 0, (core, out)
        assert _call(core, out, shape, ranks) == _lib.ERR_UNSUPPORTED, (core, out)
        assert b"not built" in _lib.lib().tnb_last_error()


def test_bad_arguments_get_their_codes():
    shape, ranks = [4, 5, 6], [1, 3, 3, 1]
    bad = [([4, 5, 6], [2, 3, 3, 1]), ([4, 5, 6], [1, 3, 3, 2]),          # boundary ranks
           ([4, 0, 6], [1, 3, 3, 1]), ([4, 5, 6], [1, 0, 3, 1]), ([4, -5, 6], [1, 3, 3, 1]),  # extent or rank below 1
           ([], [1]), ([2] * 63, [1] + [2] * 62 + [1])]                   # ndim outside [1, 62]
    for sh, rk in bad:
        assert _size(F32, F32, sh, rk) == 0, (sh, rk)
        assert _call(F32, F32, sh, rk) == _lib.ERR_INVALID, (sh, rk)
    for kw in (dict(cores=0), dict(outp=0), dict(ws=0), dict(shape_null=True), dict(ranks_null=True)):
        assert _call(F32, F32, shape, ranks, **kw) == _lib.ERR_INVALID, kw
    L = _lib.lib()
    assert L.tnb_tt_decompress_workspace_bytes(F32, F32, 3, None, _lib.i32(ranks)) == 0
    assert L.tnb_tt_decompress_workspace_bytes(F32, F32, 3, _lib.i64(shape), None) == 0
    # a result beyond 2^46 elements is refused, not mis-sized
    assert _size(F32, F32, [1 << 20] * 3, [1, 2, 2, 1]) == 0
    assert _call(F32, F32, [1 << 20] * 3, [1, 2, 2, 1]) == _lib.ERR_UNSUPPORTED


def test_no_host_synchronisation_on_the_path():
    """tnb_tt_decompress enqueues and returns: neither its driver and kernels nor the generic product they call contain
    a synchronising or allocating runtime call."""
    csrc = os.path.join(REPO, "tntorch_b200", "csrc")
    banned = re.compile(r"cuda(Stream|Device|Event)Synchronize|cudaMemcpy|cudaMalloc|cudaFree|pinned_scratch")
    for name in ("expand_tc.cuh", "gemm_generic.cuh"):
        assert not banned.search(open(os.path.join(csrc, name)).read()), name
    src = open(os.path.join(csrc, "tnb200.cu")).read()
    body = src[src.index("int tnb_tt_decompress("):]
    body = body[: body.index("\n}\n")]
    assert "tt_decompress_dispatch" in body and not banned.search(body)
