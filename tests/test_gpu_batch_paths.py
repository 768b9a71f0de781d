"""The batched dense TT-SVD (tnb_ttsvd_batch) tensor by tensor against its single calls and the fp64 oracle.

csrc/sweep.cuh ttsvd_batch_impl keeps up to `inflight` speculative sweeps in flight on internal streams, in groups of
`inflight` tensors whose workspace slice s is reused by tensor g0 + s of every group, all under TNB_FLAG_CONCURRENT,
synchronises once, and repeats the tensors whose speculation the device rejected one by one, host-driven, in slice 0.
This file
  * restates on the CPU which of its paths a batch takes (one at a time or grouped, the groups, each tensor's outcome)
    and the tensor-core Gram's split-K scratch, and checks that the batches below reach every choice;
  * runs each batch at 0, 4 and 18 reserved SMs and checks every tensor: its path against the restatement, its cores
    and ranks BITWISE against its own single call (an accepted tensor against the concurrent call at the same reserved
    SM count: the same kernels on the same grids; a repeated one against the plain call), every step against
    test_gpu_ttsvd_paths.step_oracle, ranks and relative error against oracle.tt_oracle, its input unchanged, and the
    norm the batch reports against the fp64 ||X_i||;
  * runs the benchmark's configuration (64^5 fp32, rank 32, 4 in flight, 4 reserved SMs);
  * checks the C-ABI: workspaces of exactly k slices, refusals before any launch, an empty batch, and plans sized at
    one reserved-SM count and run at another.
Run with -s to see, per tensor, the path, the largest oracle deviations and the norm shrink."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import cases as ocases
from oracle import tt_oracle as orc
from test_gpu_ttsvd_paths import (ESZ, TOL, dims, expected_flags, gram_tc_input_ok, host, make_input, on_device,
                                  project_use_tc, ranks_of, relerr, speculative, step_oracle, steps)

F32, F64 = torch.float32, torch.float64
BF16, F16, E4M3, E5M2 = torch.bfloat16, torch.float16, torch.float8_e4m3fn, torch.float8_e5m2
SXM, PCIE = 132, 114
RESERVED = (0, 4, 18)  # 18 leaves 114 usable SMs, the PCIe H100's count

# ==================================================================================================== restatement
MAX_INFLIGHT = 8  # sweep.cuh TNB_BATCH_MAX_INFLIGHT


def batch_driver(B, ws_slices, eligible):
    """(inflight, groups, one_at_a_time).  tnb200.cu:239-242: inflight = min(workspace_bytes / per_tensor_bytes, 8);
    sweep.cuh:1514-1516: one tensor at a time through the dispatcher when the batch is not speculation-eligible,
    inflight < 2 or B < 2; sweep.cuh:1527-1528, 1538-1539: else inflight clipped to B, and groups of `inflight`
    consecutive tensors (the last one partial), tensor g0 + s in slice s."""
    inflight = min(ws_slices, MAX_INFLIGHT)
    if not (B > 0 and eligible) or inflight < 2 or B < 2:
        return inflight, [], True
    inflight = min(inflight, B)
    return inflight, [list(range(g0, min(g0 + inflight, B))) for g0 in range(0, B, inflight)], False


def outcome(flags):
    """sweep.cuh:1557-1571 on a tensor's spec_check_kernel bits: 0 accepted from the in-flight sweep; bit 0 repeated
    host-driven on the exact-product Gram; otherwise (bit 4 rank below the cap, bit 5 zero unfolding) repeated
    host-driven as the single call's fallback runs it."""
    return "accepted" if flags == 0 else ("exact" if flags & 1 else "host")


TC_KC, TC_MAX_SPLIT_ITERS = 32, 512  # gram_tc.cuh


def _fold(rows, n):
    """gram_tc.cuh gram_tc_fold."""
    if n >= 128 or n < 32 or 128 % n:
        return 1
    return 128 // n if rows % (128 // n) == 0 else 1


def _ksplit(iters, cnt, sms):
    """gram_tc.cuh gram_tc_ksplit."""
    base = max(sms // cnt if cnt < sms else 1, -(-iters // TC_MAX_SPLIT_ITERS))
    ks, best, k = base, 0.0, base
    while k <= 8 * base and k <= iters and (k == base or 64 * k <= iters):
        ctas = k * cnt
        eff = ctas / (-(-ctas // sms) * sms)
        if eff > best + 0.02:
            best, ks = eff, k
        k += 1
    return min(ks, iters)


def gram_tc_scratch(rows, n, sms, max_tn=256, device_sms=None):
    """Split-K scratch bytes of the Gram of a rows x n matrix with `sms` usable SMs: gram_tc.cuh gram_tc_plan on the
    folded shape, ksplit * tiles * 128 * tn * 4.  With device_sms the factor is clamped to that of the whole device (the
    library's rule); device_sms=None gives the unclamped factor.  gram_tc_workspace_bytes = this at sms = device_sms."""
    f = _fold(rows, n)
    rows, n = rows // f, n * f
    tn = max_tn if n >= max_tn else (n + 31) // 32 * 32
    nbm, nbn = (n + 127) // 128, (n + tn - 1) // tn
    cnt = sum(1 for bm in range(nbm) for bn in range(nbn) if (bn + 1) * tn > bm * 128)
    iters = -(-rows // TC_KC)
    ks = _ksplit(iters, cnt, sms)
    if device_sms is not None and sms != device_sms:
        ks = min(ks, _ksplit(iters, cnt, device_sms))
    ips = -(-iters // ks)
    ks = -(-iters // ips)
    return -(-(ks * cnt * 128 * tn * 4) // 256) * 256


def with_slack(b):
    """tnb200.cu with_slack: the headroom a workspace query adds."""
    return b + b // 8 + (4 << 20)


def usable(sms, reserved):
    """common.cuh usable_sms."""
    return sms - min(max(reserved, 0), sms - 8)


# ==================================================================================================== batches
def _m(shape, rmax, dtype, kind="tt", **kw):
    return dict(shape=tuple(shape), rmax=[rmax] * (len(shape) - 1), dtype=dtype, kind=kind, eps=1e-14, **kw)


def _members(shape, rmax, dtype, kinds, **kw):
    """kinds: tt (accepted), low (tt with 1e-7 noise: the TF32 noise floor rejects it, bit 0), slice (a rank below the
    cap, bit 4; bit 0 too when marked), zero (bit 5), exact (a TT of rank 2 below the cap)."""
    out = []
    for k in kinds:
        if k == "low":
            out.append(_m(shape, rmax, dtype, "tt", noise=1e-7, reject=True, **kw))
        elif k == "exact":
            out.append(_m(shape, rmax, dtype, "exact", rank=2, **kw))
        else:
            out.append(_m(shape, rmax, dtype, k, **kw))
    return out


KB = (128, 128, 16, 32)  # rank 16: step 0 writes a K-blocked carry that step 1 reads
SMALL = (64, 64, 128)  # rank 8: a tensor-core step 0 for every input type, a wide step 1
BATCHES = {
    # three groups of 4, 4 and 3: each outcome in more than one group, next to the others and across a boundary
    "mixed_f32": dict(members=_members(KB, 16, F32, ["tt", "low", "slice", "zero", "tt", "zero", "low", "tt", "slice",
                                                     "low", "zero"]), inflight=4),
    "mixed_f64": dict(members=_members(SMALL, 8, F64, ["tt", "zero", "tt", "slice", "tt", "tt", "zero", "tt", "slice"]),
                      inflight=8),
    "mixed_bf16": dict(members=_members(SMALL, 8, BF16, ["tt", "zero", "tt", "slice", "tt", "tt", "zero", "tt",
                                                         "slice"]), inflight=8),
    "mixed_f16": dict(members=_members(SMALL, 8, F16, ["tt", "zero", "tt", "slice", "tt", "tt", "zero", "tt", "slice"]),
                      inflight=8),
    "mixed_e4m3": dict(members=_members(SMALL, 8, E4M3, ["tt", "zero", "tt", "slice", "tt", "tt", "zero", "tt",
                                                         "slice"]), inflight=8),
    "mixed_e5m2": dict(members=_members(SMALL, 8, E5M2, ["tt", "zero", "tt", "slice", "tt", "tt", "zero", "tt",
                                                         "slice"]), inflight=8),
    # members at 0, 4, 8 and 16 bytes past an aligned address: step 0 of the misaligned ones takes the generic Gram
    "offsets_f32": dict(members=[_m((64, 64, 32), 8, F32, off=o) for o in (0, 1, 0, 2, 4)], inflight=4),
    # a [B, ...] tensor of 840-byte samples: X[b] is misaligned for odd b
    "stacked_567_f32": dict(members=[_m((5, 6, 7), 50, F32, "randn")] * 6, inflight=8, stacked=True),
    # the reference's batch rank rule (tn.Tensor(X, batch=True)): rank = min(rmax, len(S)), a wide step
    # a zero sample keeps the caps and zero cores (before, it came back at rank 1 and tn.Tensor(X, batch=True) could
    # not stack its cores with the others')
    "batch_mode_f32": dict(members=_members((4, 8, 64), 16, F32, ["tt", "zero", "exact", "tt"]), inflight=8,
                           batch_mode=True),
    "batch_mode_f64": dict(members=_members((4, 8, 64), 16, F64, ["tt", "zero", "exact", "tt"]), inflight=8,
                           batch_mode=True),
    # one bond without a cap: not speculation-eligible, so the whole batch runs one tensor at a time
    "ineligible_f32": dict(members=[dict(c, rmax=[4, None]) for c in _members((12, 10, 8), 4, F32,
                                                                           ["tt", "zero", "tt", "tt"])], inflight=8),
}
# fp32 on the TF32 Gram: a slice's null space also sits under the noise floor (as test_gpu_ttsvd_paths' slice_f32)
BATCHES["mixed_f32"]["members"] = [dict(c, reject=True) if c["kind"] == "slice" else c
                                   for c in BATCHES["mixed_f32"]["members"]]


def _disp(case):
    """The dispatch restatement knows fp8 as e4m3; e5m2 takes the same kernels."""
    return dict(case, dtype=E4M3) if case["dtype"] == E5M2 else case


def _known_flags(case):
    """expected_flags where the data decides every bit; None where bit 0 depends on rounding the restatement does not
    model (a slice, a rank-2 TT or a zero tensor in a 16-bit or fp8 type, whose null space sits at the Gram's rounding
    level): there only bits 4 and 5 are asserted."""
    rows, rcap = dims(case["shape"], case["rmax"])
    N = len(case["shape"])
    if case["kind"] == "zero":
        want = [1] * (N + 1)
    elif case["kind"] == "slice":
        want = [1] + [min(rcap[mu], 1) for mu in range(1, N)] + [1]
    elif case["kind"] == "exact":
        want = [1] + [min(rcap[mu], case["rank"]) for mu in range(1, N)] + [1]
    else:
        want = [1] + rcap[1:N] + [1]
    f = expected_flags(case, want)
    known = case["kind"] in ("tt", "randn", "zero") or "reject" in case or case["dtype"] == F64
    return f, known


def plan_of(name, sms):
    """Per member: (eligible, flags, flags known, outcome), and the driver's choice."""
    b = BATCHES[name]
    mem = b["members"]
    elig = speculative(_disp(mem[0]), sms)
    per = []
    for c in mem:
        f, known = _known_flags(c)
        if b.get("batch_mode"):  # the rank is the cap: no bit 4; a zero sample keeps the cap too
            f &= ~16
            # the caps keep every eigenvalue of these small unfoldings, down to the fp32 solve's noise floor, where
            # rounding decides bit 0
            known = known and c["dtype"] == F64
        per.append((elig, f if elig else 0, known, outcome(f) if elig else "single"))
    inflight, groups, single = batch_driver(len(mem), b["inflight"], elig)
    return per, inflight, groups, single


def _gram0(case, sms, flags):
    """The step-0 Gram kernel of a member as the batch runs it."""
    spec = speculative(_disp(case), sms)
    accepted = spec and flags == 0
    return steps(_disp(case), sms, spec=accepted, exact=bool(flags & 1))[0]["gram"]


# ---------------------------------------------------------------------------------------------------- CPU tests
def test_batch_driver_restatement():
    """CPU: the driver restatement on the edges of tnb200.cu:242 and sweep.cuh:1516-1549."""
    assert batch_driver(11, 4, True) == (4, [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9, 10]], False)
    assert batch_driver(9, 8, True)[1] == [list(range(8)), [8]]
    assert batch_driver(5, 1, True)[2] and batch_driver(1, 8, True)[2] and batch_driver(5, 8, False)[2]
    assert batch_driver(0, 8, True)[2]
    assert batch_driver(3, 12, True)[:2] == (3, [[0, 1, 2]])
    assert batch_driver(20, 12, True)[0] == 8
    assert batch_driver(7, 2, True)[1] == [[0, 1], [2, 3], [4, 5], [6]]
    assert batch_driver(7, 3, True)[1] == [[0, 1, 2], [3, 4, 5], [6]]
    assert [outcome(f) for f in (0, 1, 17, 16, 32, 48)] == ["accepted", "exact", "exact", "host", "host", "host"]


@pytest.mark.parametrize("sms", [SXM, PCIE])
def test_batches_cover_every_driver_choice(sms):
    """CPU: the batches below and the C-ABI workspace test (k = 1, 2, 3 slices) reach every driver choice; each outcome
    appears in two groups of one batch, beside the other outcomes and on both sides of a group boundary; a member whose
    alignment changes its step-0 Gram from its neighbours'; and, for a [B, ...] tensor, that no tensor-core-eligible
    step 0 can be misaligned per sample (so the stacked batch checks the generic kernels on misaligned samples)."""
    seen = set()
    for k in (1, 2, 3):  # test_workspace_of_exactly_k_slices on mixed_f32
        seen.add(("driver", "single" if batch_driver(11, k, plan_of("mixed_f32", sms)[0][0][0])[2] else "grouped"))
    for name in BATCHES:
        per, inflight, groups, single = plan_of(name, sms)
        seen.add(("driver", "single" if single else "grouped"))
        if not per[0][0]:
            seen.add(("driver", "ineligible"))
        if len(groups) > 1 and len(groups[-1]) < inflight:
            seen.add(("driver", "partial_last_group"))
        for o in ("accepted", "exact", "host"):
            gs = [g for g in groups if any(per[i][3] == o for i in g)]
            if len(gs) >= 2 and any(len({per[i][3] for i in g}) == 3 for g in gs):
                seen.add(("outcome", o))
        for g0, g1 in zip(groups, groups[1:]):
            seen.add(("boundary", per[g0[-1]][3], per[g1[0]][3]))
        grams = {_gram0(c, sms, per[i][1]) for i, c in enumerate(BATCHES[name]["members"]) if per[i][3] == "accepted"}
        if len(grams) > 1:
            seen.add(("alignment", tuple(sorted(grams))))
    want = {("driver", d) for d in ("single", "grouped", "ineligible", "partial_last_group")}
    want |= {("outcome", o) for o in ("accepted", "exact", "host")}
    want |= {("alignment", ("generic_tall", "tc"))}
    assert not want - seen, sorted(want - seen)
    crossing = {o for k, a, b in (x for x in seen if x and x[0] == "boundary") for o in (a, b)}
    assert crossing >= {"accepted", "exact", "host"}, crossing
    # a [B, ...] sample of rows x n elements (n the last mode) is 16-byte aligned whenever the restatement lets its
    # step 0 take a tensor-core Gram or projection, so no such sample is misaligned by its neighbours
    for dt in (F32, BF16, F16, E4M3):
        for n in range(1, 513):
            for rows in (2048, 2049, 2050, 2051, 16384, 16385, 16386, 16387, 3 * 16384 + 1):
                if gram_tc_input_ok(dt, rows, n) or any(project_use_tc(dt, rows, n, r, True) for r in (1, 8, 64)):
                    assert rows * n * ESZ[dt] % 16 == 0, (dt, rows, n)
    assert 5 * 6 * 7 * 4 % 16 == 8  # the stacked batch's samples alternate between aligned and misaligned


def test_gram_scratch_restatement_and_growth():
    """CPU: the restatement reproduces the documented split-K scratch of the 64^5 step 0 (32.7 / 32.0 / 38.5 MiB at
    132 / 128 / 124 SMs: not monotone in the SM count).  Unclamped, a workspace sized at one reserved-SM count falls
    short of the scratch another count picks by more than with_slack on 40000 x 2048 (the sizing test's shape); with the
    library's clamp to the whole device's factor, every usable-SM count fits the carve."""
    MiB = 1 << 20
    assert [round(gram_tc_scratch(1 << 24, 64, s) / MiB, 1) for s in (132, 128, 124)] == [32.7, 32.0, 38.5]
    assert [round(gram_tc_scratch(40000, 2048, s) / MiB) for s in (128, 124)] == [63, 108]
    from tntorch_b200._lib import i32, i64, lib

    grow = max(gram_tc_scratch(*SIZING_SHAPE, usable(SXM, k2)) - gram_tc_scratch(*SIZING_SHAPE, usable(SXM, k1))
               for k1 in SIZING_RESERVED for k2 in SIZING_RESERVED)
    # the whole workspace the query returns (the sizing pass needs no device) is with_slack(W) for the sweep's peak W:
    # its slack, W / 8 + 4 MiB, is below what the unclamped scratch grows by
    sized = lib().tnb_ttsvd_workspace_bytes(0, 2, i64(list(SIZING_SHAPE)), i32([32]), 0)
    assert sized > 0 and grow > sized // 8 + (4 << 20), (grow / MiB, sized / MiB)
    for dev in (SXM, PCIE):
        for rows, n in ((1 << 24, 64), (1 << 18, 2048), (4096, 2048), SIZING_SHAPE, (262144, 4096), (2048, 16)):
            for mt in (256, 128):
                carve = gram_tc_scratch(rows, n, dev, mt)
                assert all(gram_tc_scratch(rows, n, s, mt, dev) <= carve for s in range(8, dev + 1)), (rows, n, mt)
    # the benchmark (4 reserved on 132) keeps its factors: no clamp applies there
    for rows, n in ((1 << 24, 64), (1 << 18, 2048), (4096, 2048)):
        assert gram_tc_scratch(rows, n, 128, 256, SXM) == gram_tc_scratch(rows, n, 128)


# ==================================================================================================== GPU helpers
def _ops():
    from tntorch_b200 import ops

    return ops


def _inputs(name):
    """Device tensors of a batch (the list run through ttsvd_batch), their fp64 values, and the [B, ...] tensor."""
    b = BATCHES[name]
    mem = b["members"]
    # make_input takes the TT rank of a "tt" member from its caps; an uncapped bond does not bound it
    X = [make_input(dict(c, rmax=[r for r in c["rmax"] if r]), 4000 + 17 * i + sum(map(ord, name)))
         for i, c in enumerate(mem)]
    if b.get("stacked"):
        st = torch.as_tensor(np.stack(X)).to(mem[0]["dtype"]).cuda()
        ds = [st[i] for i in range(len(mem))]
        return ds, [d.cpu().to(F64).numpy() for d in ds], st
    pairs = [on_device(c, x) for c, x in zip(mem, X)]
    return [p[0] for p in pairs], [p[1] for p in pairs], None


def batch_tt_svd(X, caps):
    """fp64 right-to-left TT-SVD under the reference's batch rank rule (rank = min(rmax, len(S)), no eps, no zero
    branch)."""
    shape = X.shape
    N = len(shape)
    cores = [None] * N
    C_ = X.reshape(-1, shape[-1])
    r_next = 1
    for mu in range(N - 1, 0, -1):
        M = C_.reshape(-1, shape[mu] * r_next)
        U, S, Vt = np.linalg.svd(M, full_matrices=False)
        r = min(caps[mu - 1], len(S))
        cores[mu] = Vt[:r].reshape(r, shape[mu], r_next)
        C_ = U[:, :r] * S[:r]
        r_next = r
    cores[0] = C_.reshape(1, shape[0], r_next)
    return cores


# relative shrink of ||X|| = sqrt(trace) behind a tensor-core Gram: half the trace's shrink c that DESIGN.md and
# tests/test_model.py document per type (TF32 7e-4 to 1.1e-3; bf16 9e-7, fp16 2.0e-6, e4m3 1.8e-7, e5m2 1.3e-7).
# Largest measured here on an H100 SXM (132 SMs, 700 W), printed with -s: TF32 3.5e-4, bf16 4.8e-8, fp16 9.5e-8,
# e4m3 9.4e-9, e5m2 4.9e-9
SHRINK = {F32: 5.5e-4, BF16: 4.5e-7, F16: 1e-6, E4M3: 0.9e-7, E5M2: 0.65e-7}
_REF = {}


def _check_member(name, i, case, X64, cores, single_flags, norm, sms, tol, batch_mode):
    """Oracle, gauge, chain, ranks and norm of one member; returns the printed deviations."""
    N = len(case["shape"])
    C_ = host(cores)
    gram_class = case["kind"] in ("exact", "slice")
    per, chain = step_oracle(X64, C_, case["eps"], case["rmax"], gram_class)
    rows, rcap = dims(case["shape"], case["rmax"])
    key = (name, i)
    if key not in _REF:
        _REF[key] = batch_tt_svd(X64, case["rmax"]) if batch_mode else orc.tt_svd(
            X64, ranks_tt=case["rmax"], algorithm="eig" if gram_class else "svd")
    ref = _REF[key]
    e_lib, e_ref = relerr(X64, C_), relerr(X64, ref)
    zero = case["kind"] == "zero"
    for c in C_:
        assert np.isfinite(c).all(), (name, i)
    if batch_mode:
        assert ranks_of(cores) == [1] + rcap[1:N] + [1], (name, i, ranks_of(cores))
        if zero:
            assert all(not c.any() for c in C_), (name, i)
    elif case["kind"] != "exact":
        want = [1] + [s["want"] for s in reversed(per)] + [1]
        assert ranks_of(cores) == want == ranks_of(ref), (name, i, ranks_of(cores), want, ranks_of(ref))
    for s in per:
        assert s["deficit"] <= tol["subspace"], (name, i, s)
        assert s["angle"] is None or s["angle"] <= tol["angle"], (name, i, s)
        assert zero or s["gauge"] <= tol["gauge"], (name, i, s)
    assert chain <= tol["chain"], (name, i, chain)
    assert zero or abs(e_lib - e_ref) <= tol["relerr"], (name, i, e_lib, e_ref)
    # norms[i]: ||X_i|| from the trace of step 0's Gram
    xn = float(np.linalg.norm(X64))
    g0 = _gram0(case, sms, single_flags)
    if xn == 0.0:
        assert norm == 0.0, (name, i, norm)
        shrink = 0.0
    else:
        shrink = 1.0 - norm / xn
        if g0.startswith("tc"):
            assert 0.0 <= shrink <= SHRINK[case["dtype"]], (name, i, g0, shrink)
        else:
            assert abs(shrink) <= (1e-12 if case["dtype"] == F64 else 1e-6), (name, i, g0, shrink)
    dev = max([s["deficit"] for s in per] + [0.0])
    gauge = 0.0 if zero else max(s["gauge"] for s in per)
    return (f"deficit {dev:.1e} gauge {gauge:.1e} chain {chain:.1e} relerr |diff| {abs(e_lib - e_ref):.1e} "
            f"step-0 Gram {g0} norm shrink {shrink:.1e}")


def _run_batch(name, reserved):
    ops = _ops()
    b = BATCHES[name]
    mem = b["members"]
    case0 = mem[0]
    bm = bool(b.get("batch_mode"))
    # the SM count the kernels are sized to; with Gram sides <= 256 here, speculation does not depend on it
    sms = usable(torch.cuda.get_device_properties(0).multi_processor_count, reserved)
    ds, X64s, stacked = _inputs(name)
    before = [d.clone() for d in ds]
    tol = TOL[F64 if case0["dtype"] == F64 else F32]
    per, inflight, groups, single = plan_of(name, sms)
    try:
        ops.set_reserved_sms(reserved)
        got, info = ops.ttsvd_batch(stacked if stacked is not None else ds, rmax=case0["rmax"], batch_mode=bm,
                                    inflight=b["inflight"], return_info=True)
        torch.cuda.synchronize()
        print(f"\n{name} at {reserved} reserved SMs: inflight {inflight}, groups {groups or 'one at a time'}")
        for i, (case, d, X64) in enumerate(zip(mem, ds, X64s)):
            elig, flags, known, out = per[i]
            # the single call the tensor must equal: concurrent for an accepted tensor, plain for a repeated one
            ref, rinfo = ops.ttsvd(d, rmax=case["rmax"], batch_mode=bm, concurrent=bool(info["speculative"][i]),
                                   return_info=True)
            _, pinfo = ops.ttsvd(d, rmax=case["rmax"], batch_mode=bm, return_info=True)
            sflags = pinfo["spec_flags"]
            if known:
                assert sflags == flags, (name, i, sflags, flags)
            else:
                assert sflags & 48 == flags & 48, (name, i, sflags, flags)
            assert info["speculative"][i] == int(elig and sflags == 0), (name, i, info["speculative"], sflags)
            assert info["speculative"][i] == pinfo["speculative"], (name, i)
            assert ranks_of(got[i]) == ranks_of(ref), (name, i, ranks_of(got[i]), ranks_of(ref))
            same = all(torch.equal(a, r) for a, r in zip(got[i], ref))
            msg = _check_member(name, i, case, X64, got[i], sflags, info["norms"][i], sms, tol, bm)
            print(f"  {i}: {case['kind']}{' off ' + str(case.get('off')) if case.get('off') else ''} "
                  f"{outcome(sflags) if elig else 'single'} (flags {sflags}), bitwise {same}; {msg}")
            assert same, (name, i, "batch differs from its single call")
            assert torch.equal(d, before[i]), (name, i, "input modified")
    finally:
        ops.set_reserved_sms(0)


GPU_BATCHES = list(BATCHES)


@pytest.mark.gpu
@pytest.mark.parametrize("reserved", RESERVED)
@pytest.mark.parametrize("name", GPU_BATCHES)
def test_batch_tensor_by_tensor(name, reserved):
    """Every tensor of the batch: path, bitwise equality with its single call, step oracle, ranks and relerr against
    the fp64 TT-SVD, unchanged input, and norms[i] against ||X_i||."""
    _run_batch(name, reserved)


@pytest.mark.gpu
def test_batch_constructor_with_a_zero_sample():
    """tn.Tensor(X, ranks_tt=r, batch=True) with a zero sample: every sample's cores stack at the caps, the zero
    sample's are zero and the others equal their own batch_mode calls."""
    import tntorch_b200 as tnb

    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(31)
    X = torch.randn(3, 4, 8, 64, generator=g, device="cuda")
    X[1] = 0
    t = tnb.Tensor(X, ranks_tt=16, batch=True)
    assert [tuple(c.shape) for c in t.cores] == [(3, 1, 4, 4), (3, 4, 8, 16), (3, 16, 64, 1)]
    assert all(not bool(c[1].any()) for c in t.cores)
    for b in (0, 2):
        ref = ops.ttsvd(X[b], rmax=16, batch_mode=True)
        assert all(torch.equal(c[b], r) for c, r in zip(t.cores, ref)), b


# ---------------------------------------------------------------------------------------------------- benchmark
@pytest.mark.gpu
def test_benchmark_configuration():
    """bench.py's batch: 64^5 fp32, rmax 32, 4 in flight, 4 reserved SMs; the members are the two golden tensors of
    tests/golden/full.npz and two randn tensors.  All four are accepted and each equals its single concurrent call
    bitwise, except the structured twin: its spectrum (rank 32 under 1e-2 noise) falls under the TF32 noise floor and
    it is repeated host-driven, as its single call is, and equals that call bitwise.  The golden ones meet the
    reference's ranks exactly and its relative error within 1e-5."""
    ops = _ops()
    names = ["randn64x5_r32_f32", "twin64x5_r32_f32"]
    shape = (64,) * 5
    plan_probe = ops.TTSVDPlan(shape, F32, rmax=32)
    # the four inputs, torch.randn's 4 GiB temporary, and the workspaces of the batch and of the two single plans
    need = 5 * (4 << 30) + 4 * plan_probe.ws.numel() + 2 * plan_probe.ws.numel()
    del plan_probe
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    g = np.load(__file__.rsplit("/", 1)[0] + "/golden/full.npz")
    X = torch.empty((4,) + shape, dtype=F32, device="cuda")
    for i, n in enumerate(names):
        X[i].copy_(torch.from_numpy(ocases.make_dense_big(ocases.FULL_TTSVD_CASES[n])))
    gen = torch.Generator(device="cuda").manual_seed(1234)
    for i in (2, 3):
        X[i].copy_(torch.randn(shape, generator=gen, device="cuda"))
    try:
        ops.set_reserved_sms(4)
        plan = ops.TTSVDBatchPlan(shape, F32, 4, rmax=32, inflight=4)
        got = [[c.clone() for c in cores] for cores in plan.run(X)]
        assert list(plan.spec) == [1, 0, 1, 1], list(plan.spec)
        one = {s: ops.TTSVDPlan(shape, F32, rmax=32, concurrent=bool(s)) for s in (0, 1)}
        for i in range(4):
            one[0].run(X[i])
            assert plan.spec[i] == int(one[0].info[26]), (i, list(plan.spec))
            ref = one[plan.spec[i]].run(X[i])
            assert ranks_of(got[i]) == ranks_of(ref)
            assert all(torch.equal(a, b) for a, b in zip(got[i], ref)), i
        for i, n in enumerate(names):
            err = ops.tt_relative_error(X[i], got[i])
            assert ranks_of(got[i]) == list(g[f"{n}/eig/ranks"]), n
            assert abs(err - float(g[f"{n}/eig/relerr"])) <= 1e-5, (n, err)
            print(f"{n}: relerr {err:.8f} (reference {float(g[f'{n}/eig/relerr']):.8f})")
    finally:
        ops.set_reserved_sms(0)


# ---------------------------------------------------------------------------------------------------- C-ABI
@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2, 3])
def test_workspace_of_exactly_k_slices(k):
    """A workspace of exactly k * per_tensor_bytes (k = 1: one at a time; 2, 3: grouped) gives the default plan's
    results bitwise."""
    ops = _ops()
    ds, _, _ = _inputs("mixed_f32")
    mem = BATCHES["mixed_f32"]["members"]
    shape, rmax = mem[0]["shape"], mem[0]["rmax"]
    default = ops.TTSVDBatchPlan(shape, F32, len(ds), rmax=rmax)
    want = [[c.clone() for c in cores] for cores in default.run(ds)]
    plan = ops.TTSVDBatchPlan(shape, F32, len(ds), rmax=rmax, inflight=k)
    assert plan.ws.numel() == k * plan.per_tensor_bytes
    got = plan.run(ds)
    for i in range(len(ds)):
        assert ranks_of(got[i]) == ranks_of(want[i]) and all(torch.equal(a, b) for a, b in zip(got[i], want[i])), i
    assert list(plan.spec) == list(default.spec)


def _raw_call(plan, ptrs, ws_bytes, cores_ptrs, cap, batch=None, ranks=None, norms=None, spec=None):
    ops = _ops()
    from tntorch_b200._lib import lib

    n = plan.batch if batch is None else batch
    return lib().tnb_ttsvd_batch(plan.code, ptrs, n, plan.N, plan._sh, plan._rm, 1e-14, plan.flags,
                                 ops._ptr(plan.ws), ws_bytes, cores_ptrs, cap,
                                 plan.ranks if ranks is None else ranks, plan.norms if norms is None else norms,
                                 plan.spec if spec is None else spec, ops._stream())


@pytest.mark.gpu
def test_refusals_before_any_launch_and_empty_batch():
    """A short workspace or cores capacity (TNB_ERR_WORKSPACE) and a null data pointer (TNB_ERR_INVALID) are refused
    before any launch, with the cores buffers and a guard region around them unchanged; batch = 0 returns OK and
    touches nothing."""
    ops = _ops()
    from tntorch_b200 import _lib

    shape, rmax, B = (64, 64, 32), [8, 8], 3
    plan = ops.TTSVDBatchPlan(shape, F32, B, rmax=rmax)
    xs = [torch.randn(shape, device="cuda") for _ in range(B)]
    cap = int(plan.cap)
    guard = 4096
    buf = torch.full((B * cap + 2 * guard,), 7.25, device="cuda")
    cptr = (C.c_void_p * B)(*[buf[guard + i * cap:].data_ptr() for i in range(B)])
    ptrs = (C.c_void_p * B)(*[x.data_ptr() for x in xs])
    nul = (C.c_void_p * B)(xs[0].data_ptr(), None, xs[2].data_ptr())
    ws = plan.ws.numel()
    torch.cuda.synchronize()
    for what, args, err in (("workspace", (ptrs, plan.per_tensor_bytes - 1, cptr, cap), _lib.ERR_WORKSPACE),
                            ("null data", (nul, ws, cptr, cap), _lib.ERR_INVALID),
                            ("capacity", (ptrs, ws, cptr, cap - 1), _lib.ERR_WORKSPACE)):
        n0 = ops.launch_count()
        rc = _raw_call(plan, *args)
        torch.cuda.synchronize()
        assert rc == err, (what, rc)
        assert ops.launch_count() == n0, what
        assert bool((buf == 7.25).all()), what
    ranks = (C.c_int32 * 4)(*[-5] * 4)
    norms = (C.c_double * 1)(-1.0)
    spec = (C.c_int32 * 1)(-7)
    n0 = ops.launch_count()
    assert _raw_call(plan, None, ws, None, cap, batch=0, ranks=ranks, norms=norms, spec=spec) == 0
    torch.cuda.synchronize()
    assert ops.launch_count() == n0 and list(ranks) == [-5] * 4 and norms[0] == -1.0 and spec[0] == -7
    assert bool((buf == 7.25).all())
    # and the same buffers then decompose
    assert _raw_call(plan, ptrs, ws, cptr, cap) == 0


# the shape where the split-K scratch of a plan sized at one reserved-SM count grows most when run at another (the
# restatement, test_gram_scratch_restatement_and_growth): 63 MiB at 128 usable SMs, 108 MiB at 124
SIZING_SHAPE = (40000, 2048)
SIZING_RESERVED = (0, 4, 8, 18)


@pytest.mark.gpu
def test_plan_sized_at_one_reserved_count_runs_at_another():
    """TTSVDPlan and TTSVDBatchPlan sized at k1 reserved SMs and run at k2 succeed and equal a plan sized and run at
    k2, bitwise, for k1, k2 in {0, 4, 8, 18}."""
    ops = _ops()
    gen = torch.Generator(device="cuda").manual_seed(21)
    X = torch.randn(SIZING_SHAPE, generator=gen, device="cuda")
    X2 = torch.stack([X, torch.randn(SIZING_SHAPE, generator=gen, device="cuda")])
    try:
        plans = {}
        for k in SIZING_RESERVED:
            ops.set_reserved_sms(k)
            plans[k] = (ops.TTSVDPlan(SIZING_SHAPE, F32, rmax=32),
                        ops.TTSVDBatchPlan(SIZING_SHAPE, F32, 2, rmax=32, inflight=2))
        ws = {k: (p.ws.numel(), b.ws.numel()) for k, (p, b) in plans.items()}
        print(f"\nworkspace bytes per sizing count: {ws}")
        # the split-K scratch is carved for the whole device's factor: the sizing does not depend on the reserved count
        assert len(set(ws.values())) == 1, ws
        for k2 in SIZING_RESERVED:
            ops.set_reserved_sms(k2)
            want1 = [c.clone() for c in plans[k2][0].run(X)]
            want2 = [[c.clone() for c in cores] for cores in plans[k2][1].run(X2)]
            for k1 in SIZING_RESERVED:
                got1 = plans[k1][0].run(X)
                assert all(torch.equal(a, b) for a, b in zip(got1, want1)), ("TTSVDPlan", k1, k2)
                got2 = plans[k1][1].run(X2)
                for i in range(2):
                    assert all(torch.equal(a, b) for a, b in zip(got2[i], want2[i])), ("TTSVDBatchPlan", k1, k2, i)
    finally:
        ops.set_reserved_sms(0)
