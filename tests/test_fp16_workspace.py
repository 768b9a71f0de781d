"""CPU: the dense TT-SVD's workspace for float16 input (fp16 input, fp32 carries and cores, no fp32 image of the input)
is sized without a GPU and never exceeds the fp32 workspace of the same shape and ranks."""
from oracle import cases


def test_f16_workspace_not_above_fp32():
    from tntorch_b200 import _lib

    L = _lib.lib()
    shapes = [((64,) * 5, [32] * 4)] + [(v["shape"], v["ranks_tt"]) for v in cases.TTSVD_CASES.values()
                                         if v.get("ranks_tt") is not None and "shape" in v]
    for shape, r in shapes:
        rm = r if isinstance(r, list) else [r] * (len(shape) - 1)
        sh, rc = _lib.i64(list(shape)), _lib.i32(rm)
        f32 = L.tnb_ttsvd_workspace_bytes(_lib.TNB_F32, len(shape), sh, rc, 0)
        f16 = L.tnb_ttsvd_workspace_bytes(_lib.TNB_F16, len(shape), sh, rc, 0)
        assert 0 < f16 <= f32, (shape, f16, f32)
