"""CPU: the dense TT-SVD's workspace for float8 input (e4m3 and e5m2 input, fp32 carries and cores, no fp16 or fp32 image
of the input) is sized without a GPU and never exceeds the fp16 workspace of the same shape and ranks."""
from oracle import cases


def test_f8_workspace_not_above_fp16():
    from tntorch_b200 import _lib

    L = _lib.lib()
    shapes = [((64,) * 5, [32] * 4)] + [(v["shape"], v["ranks_tt"]) for v in cases.TTSVD_CASES.values()
                                         if v.get("ranks_tt") is not None and "shape" in v]
    for shape, r in shapes:
        rm = r if isinstance(r, list) else [r] * (len(shape) - 1)
        sh, rc = _lib.i64(list(shape)), _lib.i32(rm)
        f16 = L.tnb_ttsvd_workspace_bytes(_lib.TNB_F16, len(shape), sh, rc, 0)
        for code in (_lib.TNB_F8E4M3, _lib.TNB_F8E5M2):
            f8 = L.tnb_ttsvd_workspace_bytes(code, len(shape), sh, rc, 0)
            assert 0 < f8 <= f16, (shape, code, f8, f16)


def test_f8_codes_rejected_outside_the_dense_ttsvd():
    from tntorch_b200 import _lib

    L = _lib.lib()
    sh, rk = _lib.i64([8, 8]), _lib.i32([1, 2, 1])
    for code in (_lib.TNB_F8E4M3, _lib.TNB_F8E5M2):
        assert L.tnb_tt_relative_error_workspace_bytes(code, 2, sh, rk) > 0
        assert L.tnb_gram_noise_level(code) > 0.0
    assert L.tnb_gram_noise_level(6) == 0.0
    assert L.tnb_ttsvd_workspace_bytes(6, 2, sh, _lib.i32([2]), 0) == 0  # no code past e5m2
    # 264 columns: a 16-bit Gram shape, but fp8 rows of 264 bytes are not a multiple of 16 bytes (no TMA map)
    assert L.tnb_gram_tc_f16_workspace_bytes(4096, 264) > 0 and L.tnb_gram_tc_f8_workspace_bytes(4096, 264) == 0
    assert L.tnb_gram_tc_f8_workspace_bytes(4096, 272) > 0
