"""CPU restatement of tnb_tt_multiply's shapes and envelope (csrc/tt_multiply.cuh): the rows per batch element of each
step, the chooser ttm_step_path, the launches a call makes and the workspace it asks for."""
import math

TC, F64, RANK_ALIGN, RANK_MAX, N_ODD, EXTENT, SMALL, OUT_ALIGN = range(8)
BRANCHES = {TC: "tensor cores", F64: "fp64", RANK_ALIGN: "r_k % 4 != 0", RANK_MAX: "r_k > 256", N_ODD: "N odd",
            EXTENT: "R_k < 64 or an extent >= 2^31", SMALL: "< 2^20 output elements", OUT_ALIGN: "Y not 8-byte aligned"}
EX_BN, EX_KC, EX_RS = 128, 32, 136


def step_path(f32, rows, nb, I, r, N, out_aligned=True):
    if not f32:
        return F64
    if r % 4:
        return RANK_ALIGN
    if r > 256:
        return RANK_MAX
    if N % 2:
        return N_ODD
    lim = 1 << 31
    if rows < 64 or rows >= lim or I >= lim or N >= lim:
        return EXTENT
    if nb * rows * N < (1 << 20):
        return SMALL
    if not out_aligned:
        return OUT_ALIGN
    return TC


def steps(idims, odims, ranks):
    """(R_k, i_k, r_k, N_k) per step; ranks has d + 1 entries."""
    d = len(idims)
    out = []
    for k in range(d):
        R = math.prod(idims[k + 1:]) * math.prod(odims[:k])
        out.append((R, idims[k], ranks[k], odims[k] * ranks[k + 1]))
    return out


def paths(f32, idims, odims, ranks, nb, y_aligned=True):
    st = steps(idims, odims, ranks)
    return [step_path(f32, R, nb, I, r, N, y_aligned or k + 1 < len(st)) for k, (R, I, r, N) in enumerate(st)]


def launches(f32, idims, odims, ranks, nb, y_aligned=True):
    p = paths(f32, idims, odims, ranks, nb, y_aligned)
    ntc = sum(x == TC for x in p)
    return len(p) + (ntc + 15) // 16


def _align(x):
    return (x + 255) // 256 * 256


def workspace_bytes(f32, idims, odims, ranks, nb):
    esz = 4 if f32 else 8
    st = steps(idims, odims, ranks)
    d = len(st)
    inter = max([nb * R * N for R, _, _, N in st[:-1]], default=0)
    total = (_align(inter * esz) if d > 1 else 0) + (_align(inter * esz) if d > 2 else 0)
    for R, I, r, N in st:
        if step_path(f32, R, nb, I, r, N) == TC:
            kcr = -(-r // 8) * 8 if r <= EX_KC else EX_KC
            total += _align(-(-N // EX_BN) * I * -(-r // EX_KC) * 2 * kcr * EX_RS * 4)
    return max(total, 256)
