"""CPU: tnb_tt_multiply is sized without a GPU and its size is restated from the shapes (two ping-pong intermediates of
the largest step output and the TF32 images of the tensor-core steps' cores, never M or a copy of X), unsupported
dtypes size to 0 and are refused with TNB_ERR_UNSUPPORTED, malformed arguments get their codes before anything is
launched, and no host synchronisation is on the path (checked on the source)."""
import ctypes
import math
import os
import re

import ttm_model as tm
from tntorch_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64 = _lib.TNB_F32, _lib.TNB_F64

SHAPES = [([13], [11], [1, 1], 127), ([8, 16], [64, 4], [1, 16, 1], 4097), ([8] * 3, [8] * 3, [1, 16, 16, 1], 4097),
          ([8] * 3, [8] * 3, [1, 4, 12, 1], 4097), ([4, 8, 8], [8, 8, 4], [1, 36, 36, 1], 127),
          ([4, 2, 8], [8, 2, 3], [1, 256, 2, 1], 4097), ([8] * 4, [8] * 4, [1, 32, 32, 32, 1], 16384),
          ([8] * 4, [8] * 4, [1, 16, 16, 16, 1], 8192), ([4] * 5, [4] * 5, [1] + [8] * 4 + [1], 65536),
          ([2, 3, 1, 5, 2, 2], [3, 1, 2, 2, 5, 1], [1, 3, 7, 5, 4, 2, 1], 127), ([11, 3], [23, 2], [1, 50, 1], 30)]


def _size(dtype, idims, odims, ranks, nb):
    return _lib.lib().tnb_tt_multiply_workspace_bytes(dtype, len(idims), _lib.i64(idims), _lib.i64(odims),
                                                      _lib.i32(ranks), nb)


def _call(dtype, idims, odims, ranks, nb, cores=1, x=1, y=1, ws=1, ws_bytes=1 << 40, nulls=()):
    """The run entry with dummy non-null pointers: every check below fails before anything is dereferenced."""
    d = len(idims)
    buf = (ctypes.c_double * 8)()
    ptrs = (ctypes.c_void_p * max(d, 1))(*([ctypes.addressof(buf)] * max(d, 1)))
    p = ctypes.c_void_p(ctypes.addressof(buf))
    return _lib.lib().tnb_tt_multiply(dtype, ptrs if cores else None, d, None if "i" in nulls else _lib.i64(idims),
                                      None if "o" in nulls else _lib.i64(odims), None if "r" in nulls else _lib.i32(ranks),
                                      p if x else None, nb, p if y else None, p if ws else None, ws_bytes, None)


def test_workspace_is_restated_from_the_shapes():
    for idims, odims, ranks, nb in SHAPES:
        for dt in (F32, F64):
            assert _size(dt, idims, odims, ranks, nb) == tm.workspace_bytes(dt == F32, idims, odims, ranks, nb), (idims, ranks, dt)


def test_workspace_never_holds_m_or_a_copy_of_x():
    """Without tensor-core steps (fp64) the workspace is the two intermediates alone; it never grows with I * O."""
    for idims, odims, ranks, nb in SHAPES:
        st = tm.steps(idims, odims, ranks)
        inter = max([nb * R * N for R, _, _, N in st[:-1]], default=0)
        assert _size(F64, idims, odims, ranks, nb) <= max(256, 2 * (inter * 8 + 255))
    # 8^4 -> 8^4 at rank 16: M would be 4096^2 fp32 (64 MB) and X 128 MB; the workspace is the two intermediates
    idims, odims, ranks, nb = [8] * 4, [8] * 4, [1, 16, 16, 16, 1], 8192
    assert _size(F32, idims, odims, ranks, nb) < 2 * nb * 512 * 128 * 4 + (1 << 20)


def test_supported_calls_never_size_to_zero():
    for dt in (F32, F64):
        assert _size(dt, [1], [1], [1, 1], 1) >= 256
        assert _size(dt, [2] * 20 + [1] * 44, [1] * 64, [1] * 65, 1) >= 256


def test_unsupported_dtypes_size_to_zero_and_are_refused():
    for dt in (_lib.TNB_BF16, _lib.TNB_F16, _lib.TNB_F8E4M3, _lib.TNB_F8E5M2, 7, -1):
        assert _size(dt, [8, 8], [8, 8], [1, 4, 1], 16) == 0
        assert _call(dt, [8, 8], [8, 8], [1, 4, 1], 16) == _lib.ERR_UNSUPPORTED
        assert b"not built" in _lib.lib().tnb_last_error()


def test_malformed_arguments_get_their_codes():
    idims, odims, ranks = [4, 5, 6], [3, 2, 2], [1, 3, 3, 1]
    invalid = [(idims, odims, [2, 3, 3, 1], 8), (idims, odims, [1, 3, 3, 2], 8),      # boundary ranks
               ([4, 0, 6], odims, ranks, 8), (idims, [3, -2, 2], ranks, 8), (idims, odims, [1, 0, 3, 1], 8),
               (idims, odims, ranks, 0), (idims, odims, ranks, -3),                   # non-positive dims or batch
               ([], [], [1], 8), ([2] * 65, [1] * 65, [1] * 66, 8)]                   # d outside [1, 64]
    for i, o, r, nb in invalid:
        assert _size(F32, i, o, r, nb) == 0, (i, o, r, nb)
        assert _call(F32, i, o, r, nb) == _lib.ERR_INVALID, (i, o, r, nb)
    for kw in (dict(cores=0), dict(x=0), dict(y=0), dict(ws=0), dict(nulls="i"), dict(nulls="o"), dict(nulls="r")):
        assert _call(F32, idims, odims, ranks, 8, **kw) == _lib.ERR_INVALID, kw
    L = _lib.lib()
    assert L.tnb_tt_multiply_workspace_bytes(F32, 3, None, _lib.i64(odims), _lib.i32(ranks), 8) == 0
    assert L.tnb_tt_multiply_workspace_bytes(F32, 3, _lib.i64(idims), _lib.i64(odims), None, 8) == 0
    # sizes that overflow: refused, not mis-sized
    big = [([1 << 24] * 2, [1 << 24] * 2, [1, 1, 1], 1), ([64], [64], [1, 1], 1 << 31), ([1 << 20], [1 << 20], [1, 1], 1 << 27)]
    for i, o, r, nb in big:
        assert _size(F32, i, o, r, nb) == 0, (i, o, r, nb)
        assert _call(F32, i, o, r, nb) == _lib.ERR_UNSUPPORTED, (i, o, r, nb)


def test_no_host_synchronisation_on_the_path():
    csrc = os.path.join(REPO, "tntorch_b200", "csrc")
    banned = re.compile(r"cuda(Stream|Device|Event)Synchronize|cudaMemcpy|cudaMalloc|cudaFree|pinned_scratch")
    for name in ("tt_multiply.cuh", "expand_tc.cuh", "project_tc.cuh"):
        assert not banned.search(open(os.path.join(csrc, name)).read()), name
    src = open(os.path.join(csrc, "tnb200.cu")).read()
    body = src[src.index("int tnb_tt_multiply("):]
    body = body[: body.index("\n}\n")]
    assert "tt_multiply_dispatch" in body and not banned.search(body)
    # the Python call: no .item(), .cpu(), .tolist() or synchronize on the device path
    ops = open(os.path.join(REPO, "tntorch_b200", "ops.py")).read()
    fn = ops[ops.index("def tt_multiply("):]
    assert not re.search(r"\.item\(|\.cpu\(|\.tolist\(|synchronize|\.numpy\(", fn)


def test_chooser_restatement_matches_the_source():
    """The constants of the CPU restatement are the header's."""
    src = open(os.path.join(REPO, "tntorch_b200", "csrc", "tt_multiply.cuh")).read()
    assert "TTM_TC_MAX_R = 256;" in src and "TTM_TC_MIN_ROWS = 64;" in src and "TTM_TC_MIN_ELEMS = (int64_t)1 << 20;" in src
    assert tm.step_path(True, 64, 4097, 8, 16, 4) == tm.TC
    assert tm.step_path(True, 63, 1 << 20, 8, 16, 4) == tm.EXTENT
    assert math.prod([1]) == 1
