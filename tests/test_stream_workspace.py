"""CPU: the workspace of the streamed dense TT-SVD (tnb_ttsvd_stream_workspace_bytes) and its refusals, sized without a
GPU; the chunk plan and tn.Tensor's stream-or-copy rule restated (stream_model.py), with coverage tests."""
import numpy as np

from oracle import cases
import stream_model as sm


def _ws(code, shape, r, chunk=0):
    from tntorch_b200 import _lib

    rm = r if isinstance(r, list) else [r] * max(len(shape) - 1, 1)
    return _lib.lib().tnb_ttsvd_stream_workspace_bytes(code, len(shape), _lib.i64(list(shape)), _lib.i32(rm), chunk, 0)


def test_larger_than_device_tensors_fit_80GB():
    from tntorch_b200 import _lib

    for shape, r in (((128,) * 5, 16), ((32,) * 7, 8)):  # 128 GiB of fp32 each
        assert 4 * int(np.prod(shape)) == 128 << 30
        b = _ws(_lib.TNB_F32, shape, r)
        assert 0 < b < 80e9, (shape, b)
        carry = 4 * int(np.prod(shape[:-1])) * r
        assert b > carry  # the step-0 carry lives in the workspace, the input never does


def test_below_device_call_plus_input_for_every_capped_case():
    from tntorch_b200 import _lib

    L = _lib.lib()
    for name, v in cases.TTSVD_CASES.items():
        if v.get("ranks_tt") is None or "shape" not in v:
            continue
        code, esz = (_lib.TNB_F32, 4) if v["dtype"] == "float32" else (_lib.TNB_F64, 8)
        shape, r = v["shape"], v["ranks_tt"]
        rm = r if isinstance(r, list) else [r] * (len(shape) - 1)
        dev = L.tnb_ttsvd_workspace_bytes(code, len(shape), _lib.i64(list(shape)), _lib.i32(rm), 0)
        assert _ws(code, shape, r) < dev + int(np.prod(shape)) * esz, name


def test_refusals():
    from tntorch_b200 import _lib

    L = _lib.lib()
    assert _ws(_lib.TNB_F32, (4, 100), 3) == 0 and b"wide" in L.tnb_last_error()
    assert _ws(_lib.TNB_F32, (100,), [1]) == 0 and b"mode" in L.tnb_last_error()
    assert _ws(_lib.TNB_F32, (32,) * 7, 32) == 0 and b"carry" in L.tnb_last_error()  # carry as large as the input
    assert _ws(6, (64, 64, 64), 8) == 0  # no code past e5m2
    for code in (_lib.TNB_F32, _lib.TNB_F64, _lib.TNB_BF16, _lib.TNB_F16, _lib.TNB_F8E4M3, _lib.TNB_F8E5M2):
        assert _ws(code, (32,) * 5, 16) > 0


def test_ring_follows_the_chunk_budget():
    """the ring is two chunks of the planned size, or one chunk holding the whole tensor (the rest of the sweep reuses
    its memory, so the difference is the ring's less what the sweep needs beyond a small ring)."""
    from tntorch_b200 import _lib

    shape, r = (64,) * 5, 32
    one = _ws(_lib.TNB_F32, shape, r, 8 << 30)
    small = _ws(_lib.TNB_F32, shape, r, 64 << 20)
    assert (3 << 30) < one - small < 4 << 30


# ---- the chunk plan ------------------------------------------------------------------------------------------------
# (rows, n, row_bytes, chunk_bytes, proj_tc, kb_inner) -> (chunk_rows, nchunks, last_rows): the GPU tests' shapes and budgets
PLANS = {
    "fp32_32x5_r16_one": ((32 ** 4, 32, 128, 0, True, 32), (32 ** 4, 1, 32 ** 4)),
    "fp32_32x5_r16_two": ((32 ** 4, 32, 128, 2 ** 26 + 1, True, 32), (2 ** 19, 2, 2 ** 19)),
    "fp32_32x5_r16_ragged7": ((32 ** 4, 32, 128, 2 ** 27 * 2 // 13, True, 32), (161280, 7, 80896)),
    "fp32_32x5_r16_minimum": ((32 ** 4, 32, 128, 1, True, 32), (16384, 64, 16384)),
    "fp32_32x5_r8_minimum": ((32 ** 4, 32, 128, 1, True, 0), (16384, 64, 16384)),
    "bf16_32x5_r16_64th": ((32 ** 4, 32, 64, 2 ** 20, False, 0), (16384, 64, 16384)),
    "fp64_32x5_ragged7": ((32 ** 4, 32, 256, 2 ** 28 * 2 // 13, False, 0), (161312, 7, 80704)),
    "twin64x5_64MiB": ((64 ** 4, 64, 256, 64 << 20, True, 64), (262144, 64, 262144)),
    "short_last_piece_joins": ((40000, 32, 128, 1, True, 0), (16384, 2, 23616)),
    "short_last_piece_joins_2": ((50000, 32, 128, 1, True, 0), (16384, 3, 17232)),
    "cfg1_thirds": ((4096, 16, 64, 4096 * 64 // 3, False, 0), (1360, 4, 16)),
    "two_modes_thirds": ((40, 30, 240, 40 * 30 * 8 // 3, False, 0), (32, 1, 40)),  # chunks of >= 30 rows: the n x n Gram
    "lownoise_16x5_thirds": ((16 ** 4, 16, 64, 16 ** 5 * 4 // 3, False, 0), (21840, 4, 16)),
}


def test_chunk_plan_restatement():
    for name, (args, want) in PLANS.items():
        unit, min_rows, chunk_rows, n, last = sm.chunk_plan(*args)
        assert (chunk_rows, n, last) == want, (name, (chunk_rows, n, last))
        rows = args[0]
        assert (n - 1) * chunk_rows + last == rows and chunk_rows % unit == 0
        assert n == 1 or last >= min_rows


def test_chunk_plans_cover_every_branch():
    seen = set()
    for args, _ in PLANS.values():
        unit, min_rows, chunk_rows, n, last = sm.chunk_plan(*args)
        seen.add("kblocked_unit" if args[5] else "unit16")
        seen.add("tc_minimum" if min_rows == sm.PROJ_TC_MIN_ROWS else "columns_minimum")
        seen.add("single" if n == 1 else "ragged" if last != chunk_rows else "even")
        if n < -(-args[0] // chunk_rows):
            seen.add("joined")
        seen.add("default_budget" if args[3] == 0 else "budget")
    assert seen == {"kblocked_unit", "unit16", "tc_minimum", "columns_minimum", "single", "ragged", "even", "joined",
                    "default_budget", "budget"}, seen


# ---- tn.Tensor's stream-or-copy rule -----------------------------------------------------------------------------------
RULE = [  # (input bytes, device-call workspace, free bytes)
    (128 << 30, 3 << 30, 79 << 30), (4 << 30, 3 << 30, 79 << 30), (70 << 30, 9 << 30, 79 << 30),
    (70 << 30, (9 << 30) + 1, 79 << 30), (1 << 20, 0, 1 << 20), (1 << 20, 1, 1 << 20),
]


def test_stream_rule_restatement():
    from tntorch_b200 import ops

    for a in RULE:
        assert ops.stream_instead_of_copy(*a) == sm.streams(*a) == (a[0] + a[1] > a[2]), a


def test_stream_rule_cases_cover_both_sides_and_the_boundary():
    outcomes = {sm.streams(*a) for a in RULE}
    assert outcomes == {True, False}
    assert any(a[0] + a[1] == a[2] for a in RULE) and any(a[0] + a[1] == a[2] + 1 for a in RULE)
