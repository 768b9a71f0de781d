"""Tucker rounding, tn.round and the ranks_tucker / eps constructors path by path against the fp64 oracle.

Paths (tensor.py round_tucker, round, the Tensor(X, eps=) and Tensor(X, ranks_tucker=[, ranks_tt=]) branches): per mode,
the Householder QR of the (r0 r1) x S unfolding (tall: k = S, wide: k = r0 r1), the split of the I x k factor by
truncated_svd (left Gram when I <= k, right Gram with the gauge repair when I > k; the eigensolver tsvd_eig picks by
L = min(I, k)), the rule (eps, rmax or both), and whether the mode had a factor or a CP core before.  Per case, on the
values of the device input widened to fp64: (a) the Tucker and TT ranks (exact where the oracle's margin is large, else
true rank <= r <= cap), (b) the relative error against the oracle's, (c) relerr <= eps plus noise for the eps rules,
(d) each factor's subspace on gapped modes, (e) |U^T U - I| and the right gauge of cores 1..N-1, (f) tucker_core() and
decompress_tucker_factors() against the oracle's contraction, (g) the inputs of tn.round_tucker / tn.round unchanged,
(h) the eigensolver kernels the restatement names (torch.profiler), and what round_tucker passes to truncated_svd (the
budget eps / sqrt(len(dim)), rmax, I and k) and what tn.round passes to round_tucker ((1 + eps) / (1 + reached) - 1).
Also: CP on a Tucker core as a composition, orthogonalisation of batched TT, CP and TT-Tucker cores, and the refusals
(a refused rounding leaves the tensor as it was).

CP cores: the reference's round_tucker turns the CP factors of `dim` into [R, I, R] cores one by one (tensor.py:1943),
so its first and last TT ranks become R; this package converts them with the whole-tensor rule of round_tt (first
[1, I, R], last [R, I, 1]), the same tensor with boundary ranks 1.  The oracle is therefore run on the converted cores
for the device comparison; the reference's own Tucker ranks are checked against the golden.
Run with -s to see the measured deviations."""
import contextlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import cases
from oracle import tt_oracle as orc
from test_gpu_arith_paths import oracle_rank, principal_sin, tsvd_adaptive_block, tsvd_eig, tsvd_form, tsvd_side

F32, F64 = torch.float32, torch.float64
EPS64 = float(np.finfo(np.float64).eps)
GOLD = os.path.join(os.path.dirname(__file__), "golden", "tucker.npz")
CASES = {**cases.TUCKER_CASES, **cases.TUCKER_PATH_CASES}

# Bounds, each at most 10x the largest value measured on an H100 SXM (132 SMs, 700 W) over the cases here, which is quoted
# per entry (printed with -s as "MEASURED <type> <key> <value>").
#   relerr:  (b) |relerr(device) - relerr(oracle)| beyond the slack of the modes decided at the noise
#   eps_noise: (c) relerr - eps against the tensor decomposed (for a 16- or 8-bit input, its own values)
#   angle:   (d) sin of the largest principal angle           gauge:     (e) |U^T U - I| and |C C^T - I|
#   compose: (f) max |device - oracle| / max |oracle|         ortho:     |abs(device core) - abs(oracle core)| / max
#   ortho_dense: orthogonalisation changes the tensor by this much (relative)
TOL = {
    F64: dict(relerr=5e-13,            # 4.98e-14
              eps_noise=1e-12,         # 0
              angle=4e-7,              # 4e-8 (dense_analytic128_tucker3: its exact TT drops directions at the noise floor)
              gauge=1.1e-12,           # 1.03e-13
              compose=6.1e-15,         # 6.03e-16
              ortho=1.5e-14,           # 1.48e-15
              ortho_dense=9.2e-15),    # 9.16e-16
    F32: dict(relerr=3.7e-6,           # 3.62e-7
              eps_noise=1e-6,          # 0
              angle=1.8e-6,            # 1.72e-7
              gauge=1.3e-6,            # 1.23e-7
              compose=4.1e-6,          # 4.09e-7
              ortho=1.9e-6,            # 1.91e-7
              ortho_dense=1.9e-6),     # 1.87e-7
    torch.bfloat16: dict(relerr=1.9e-7,        # 1.81e-8
                         eps_noise=1e-6,       # 0
                         angle=9.2e-7,         # 9.2e-8
                         gauge=9.8e-7,         # 9.78e-8
                         compose=3.6e-6),      # 3.59e-7
    torch.float8_e4m3fn: dict(relerr=3.1e-6,   # 3.1e-7
                              eps_noise=1e-6,  # 0
                              angle=1.2e-6,    # 1.18e-7
                              gauge=3.6e-6,    # 3.59e-7
                              compose=3.6e-6), # 3.51e-7
}
LOW = (torch.bfloat16, torch.float8_e4m3fn)


def bound(key, dtype, value):
    print(f"\nMEASURED {str(dtype)[6:]} {key} {value:.3g}")
    tol = TOL[dtype][key]
    assert value <= tol, (key, str(dtype), value, tol)


# ==================================================================================================== inputs and oracle
def case_input(c, dtype):
    """The case's input on the device in `dtype` and the same values widened to fp64: (dense or None, cores, Us)."""
    if c["kind"] == "dense":
        X = torch.as_tensor(cases.make_dense(dict(c["spec"], dtype="float64"))).to(dtype).cuda()
        return X, None, None
    cores, Us = cases.make_tucker_input(dict(c["spec"], dtype="float64"))
    cd = [torch.as_tensor(x).to(dtype).cuda() for x in cores]
    Ud = [None if U is None else torch.as_tensor(U).to(dtype).cuda() for U in Us]
    return None, cd, Ud


def widen(x):
    return None if x is None else x.double().cpu().numpy()


def oracle_case(c, X64=None, cores64=None, Us64=None):
    """The case on the oracle: (cores, Us, round_tucker's info or None, reached or None).  CP cores are converted with
    the whole-tensor rule first (module docstring)."""
    if c["kind"] == "dense":
        if "eps" in c:
            cores, Us, reached, info = orc.tucker_eps(X64, c["eps"])
            return cores, Us, info, reached
        cores, Us, info = orc.tucker_from_dense(X64, c["ranks_tucker"], c.get("ranks_tt"))
        return cores, Us, info, None
    cores, Us = [x.copy() for x in cores64], [None if U is None else U.copy() for U in Us64]
    orc.cp_to_tt(cores)
    if "round_tucker" in c:
        return cores, Us, orc.round_tucker(cores, Us, **c["round_tucker"]), None
    reached, info = orc.round(cores, Us, **c["round"])
    return cores, Us, info, reached


def eps_rule(c):
    """The relative error the case's call promises not to exceed, or None."""
    if c["kind"] == "dense":
        return c.get("eps")
    if "round_tucker" in c:
        # with `dim` a subset every mode is still split, each under eps / sqrt(len(dim)): no promise (the reference's
        # tt_dim_subset ends at 0.2016 for eps = 0.2)
        kw = c["round_tucker"]
        return kw.get("eps") if kw.get("rmax") is None and "eps" in kw and "dim" not in kw else None
    kw = c["round"]
    return kw["eps"] if kw.get("rmax") is None else None


# ==================================================================================================== CPU part
def mode_plan(c):
    """Per mode, in the order round_tucker visits them, what it runs: the QR shape and k, the truncated_svd side, form
    and eigensolver, the rule, and whether the mode had a factor / a CP core.  Taken from the fp64 oracle's run of the
    case (the ranks of later modes depend on the earlier decisions)."""
    X, cores, Us = None, None, None
    if c["kind"] == "dense":
        X = cases.make_dense(dict(c["spec"], dtype="float64"))
    else:
        cores, Us = cases.make_tucker_input(dict(c["spec"], dtype="float64"))
    info = oracle_case(c, X, cores, Us)[2] or []
    was_cp = [x.ndim == 2 for x in cores] if cores is not None else []
    plan = []
    for m in info:
        I, k, rmax = m["I"], m["k"], m["rmax"]
        rule = "both" if (rmax is not None and m["eps"] > 1e-13) else ("rmax" if rmax is not None else "eps")
        eig = tsvd_eig(I, k, rmax)
        if eig == "adaptive" and tsvd_adaptive_block(m["rank"]) is None:  # the rule's rank passes 240: refused
            eig = "refused"
        plan.append(dict(mu=m["mu"], qr="tall" if m["rows"] >= m["S"] else "wide", k=k, I=I, side=tsvd_side(I, k),
                         form=tsvd_form(I, k, True), eig=eig, rule=rule, had_U=m["had_U"],
                         cp=was_cp[m["mu"]] if was_cp else False, N=len(info)))
    return plan


# refused: round_tucker of a (24, 300, 24) TT of ranks 24 reaches mode 1 with L = 300 and a numerical rank of 300 after
# mode 2 was cut to 20; tn.round(eps=1e-6) reaches it the same way after the TT rounding
# (the reference completes both)
REFUSED = {
    "round_tucker_after_a_cut": dict(kind="tt", spec=dict(shape=(24, 300, 24), rank=24, seed=91, dtype="float64"),
                                     round_tucker=dict(rmax=[None, None, 20])),
    "round_after_round_tt": dict(kind="tt", spec=dict(shape=(24, 300, 24), rank=24, seed=92, dtype="float64"),
                                 round=dict(eps=1e-6)),
}


def test_mode_plan_reaches_every_path():
    seen = {k: set() for k in ("qr", "side", "form", "eig", "rule")}
    cp_pos, had_U = set(), False
    big = False
    for c in list(CASES.values()) + list(REFUSED.values()):
        for p in mode_plan(c):
            for k in seen:
                seen[k].add(p[k] if k != "form" else (p["side"],) + p["form"])
            if p["cp"]:
                cp_pos.add("first" if p["mu"] == 0 else ("last" if p["mu"] == p["N"] - 1 else "middle"))
            had_U |= p["had_U"]
            big |= p["eig"] in ("chfsi", "adaptive") and p["I"] > 256 and p["k"] > 256
    assert [p["eig"] for r in REFUSED.values() for p in mode_plan(r)].count("refused") == len(REFUSED)
    assert seen["qr"] == {"tall", "wide"}
    assert seen["side"] == {"left", "right"}
    assert seen["form"] == {("left", "left", False), ("right", "left", True)}  # r0 r1 >= I: left Gram; else the repair
    assert seen["eig"] == {"jac2_f64", "jac2_mixed", "onesided_smem", "onesided_gmem", "chfsi", "adaptive", "refused"}
    assert seen["rule"] == {"eps", "rmax", "both"}
    assert cp_pos == {"first", "middle", "last"} and had_U and big


# the seven cases the golden file had before it was extended: regenerating it must leave them bitwise as they were
OLD_GOLDEN = {
    "dense_analytic128_eps": ([1, 4, 6, 1], [4, 5, 6], "0x1.17da03b251002p-17"),
    "dense_analytic128_tucker3": ([1, 9, 3, 1], [3, 3, 3], "0x1.0c99eecc8cb0ep-11"),
    "dense_randn16x3_tucker3": ([1, 9, 3, 1], [3, 3, 3], "0x1.ef93d54917423p-1"),
    "dense_twin_eps": ([1, 4, 4, 4, 4, 1], [4, 10, 8, 9, 4], "0x1.0aa720f7728d1p-20"),
    "tt_round_eps": ([1, 6, 7, 7, 6, 1], [6, 10, 10, 10, 6], "0x1.bcdb185a36a41p-4"),
    "tt_round_tucker_eps": ([1, 6, 6, 6, 1], [6, 15, 15, 6], "0x1.dcdd8cef1d6a5p-4"),
    "tt_round_tucker_rmax": ([1, 5, 5, 4, 1], [4, 4, 4, 4], "0x1.7a28f9597c999p-1"),
}


def test_old_golden_keys_unchanged():
    g = np.load(GOLD)
    for name, (rt, ru, e) in OLD_GOLDEN.items():
        assert g[f"{name}/ranks_tt"].tolist() == rt and g[f"{name}/ranks_tucker"].tolist() == ru
        assert float(g[f"{name}/relerr"]).hex() == e, name


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference(name):
    """The oracle on the case's own input (CP cores as the reference converts them) against the reference's run."""
    g = np.load(GOLD)
    c = CASES[name]
    if c["kind"] == "dense":
        X = cases.make_dense(c["spec"])
        out = oracle_case(c, X)
        cores, Us, dense = out[0], out[1], X
    else:
        cores, Us = cases.make_tucker_input(c["spec"])
        dense = orc.tucker_full([x.copy() for x in cores], Us)
        cores, Us = [x.copy() for x in cores], list(Us)
        if "round_tucker" in c:
            orc.round_tucker(cores, Us, **c["round_tucker"])
        else:
            orc.round(cores, Us, **c["round"])
    tt = orc.cp_to_tt(list(cores))
    assert [tt[0].shape[0]] + [x.shape[2] for x in tt] == g[f"{name}/ranks_tt"].tolist()
    assert [x.shape[1] for x in tt] == g[f"{name}/ranks_tucker"].tolist()
    err = float(np.linalg.norm(orc.tucker_full(cores, Us) - dense) / np.linalg.norm(dense))
    ref = float(g[f"{name}/relerr"])
    assert abs(err - ref) <= (2e-5 if c["spec"].get("dtype") == "float32" else 1e-9) * max(ref, 1e-6), (err, ref)


def test_oracle_cp_to_tt_and_factor_orthogonalize_keep_the_tensor():
    rng = np.random.default_rng(3)
    cores = [rng.standard_normal((s, 4)) for s in (5, 6, 7)]
    Us = [rng.standard_normal((I, s)) for I, s in zip((8, 9, 10), (5, 6, 7))]
    want = np.einsum("ar,br,cr->abc", *[U @ c for U, c in zip(Us, cores)])
    assert np.allclose(orc.tucker_full(cores, Us), want, atol=1e-12 * np.abs(want).max())
    tt = orc.cp_to_tt(list(cores))
    assert [x.shape for x in tt] == [(1, 5, 4), (4, 6, 4), (4, 7, 1)]
    for mu in range(3):
        cs, us = list(cores), list(Us)
        orc.factor_orthogonalize(cs, us, mu)
        assert np.allclose(us[mu].T @ us[mu], np.eye(us[mu].shape[1]), atol=1e-13)
        assert np.allclose(orc.tucker_full(cs, us), want, atol=1e-12 * np.abs(want).max())


# ==================================================================================================== GPU part
@contextlib.contextmanager
def spy():
    """Records what round_tucker passes to ops.truncated_svd and what Tensor.round / the eps constructor pass to
    round_tucker (with the dense tensor at that moment)."""
    import tntorch_b200 as tnb
    from tntorch_b200 import ops

    calls = dict(tsvd=[], round_tucker=[])
    orig_tsvd, orig_rt = ops.truncated_svd, tnb.Tensor.round_tucker

    def tsvd(M, *a, **kw):
        calls["tsvd"].append(dict(I=M.shape[0], k=M.shape[1], eps=kw.get("eps"), rmax=kw.get("rmax")))
        return orig_tsvd(M, *a, **kw)

    def rt(self, eps=1e-14, *a, **kw):
        calls["round_tucker"].append(dict(eps=eps, dense=self.torch().double().cpu().numpy()))
        return orig_rt(self, eps, *a, **kw)

    ops.truncated_svd, tnb.Tensor.round_tucker = tsvd, rt
    try:
        yield calls
    finally:
        ops.truncated_svd, tnb.Tensor.round_tucker = orig_tsvd, orig_rt


def device_case(c, X, cores, Us):
    import tntorch_b200 as tnb

    if c["kind"] == "dense":
        kw = {k: c[k] for k in ("ranks_tucker", "ranks_tt", "eps") if k in c}
        return tnb.Tensor(X, **kw)
    t = tnb.Tensor(cores, Us=Us if Us[0] is not None else None)
    if "round_tucker" in c:
        return tnb.round_tucker(t, **c["round_tucker"])
    return tnb.round(t, **c["round"])


def run_params():
    out = []
    for name, c in CASES.items():
        if name.startswith("dense_analytic128"):  # 128^3: once, in fp64
            out.append((name, F64))
            continue
        out += [(name, F64), (name, F32)]
        if c["kind"] == "dense":
            out += [(name, dt) for dt in LOW]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name,dtype", run_params(), ids=[f"{n}-{str(d)[6:]}" for n, d in run_params()])
def test_case_against_oracle(name, dtype):
    c = CASES[name]
    g = np.load(GOLD)
    X, cores, Us = case_input(c, dtype)
    before = None if X is not None else ([x.clone() for x in cores], [None if U is None else U.clone() for U in Us])
    with spy() as calls:
        t = device_case(c, X, cores, Us)
    torch.cuda.synchronize()
    # (g) the inputs of tn.round_tucker / tn.round are left as they were
    if before is not None:
        assert all(torch.equal(a, b) for a, b in zip(cores, before[0]))
        assert all((a is None and b is None) or torch.equal(a, b) for a, b in zip(Us, before[1]))
    X64 = widen(X)
    c64 = None if cores is None else [widen(x) for x in cores]
    U64 = None if Us is None else [widen(U) for U in Us]
    dense = X64 if X64 is not None else orc.tucker_full(c64, U64)
    ocores, oUs, info, reached = oracle_case(c, X64, c64, U64)
    nrm = float(np.linalg.norm(dense))
    e_orc = float(np.linalg.norm(orc.tucker_full(ocores, oUs) - dense)) / nrm
    dc = [widen(x) for x in t.cores]
    dU = [widen(U) for U in t.Us]
    e_dev = float(np.linalg.norm(orc.tucker_full(dc, dU) - dense)) / nrm
    # the resolution of the tail sums, relative to the trace: fp64, or fp32 (a 16- or 8-bit input is decomposed into fp32
    # cores; the sweep's projections are fp32-accurate 3xTF32 products, its TF32 Grams decide ranks under the accept rule)
    noise = EPS64 if dtype == F64 else 1e-9
    # what round_tucker ran, mode by mode, against the oracle's (I, k, budget, rmax); the leftover budget of tn.round /
    # Tensor(eps=) against (1 + eps) / (1 + reached) - 1 with reached measured on the tensor round_tucker was given
    if info is not None:
        assert len(calls["round_tucker"]) >= 1
        got = calls["tsvd"][-len(info):]
        assert [(m["I"], m["rmax"]) for m in got] == [(m["I"], m["rmax"]) for m in info], (got, info)
        # k: the exact TT of a dense input (ops.ttsvd, eps = 0) drops the directions at its eigensolver's noise floor
        # that _full_rank_tt keeps, so its k may be smaller there
        assert all(m["k"] == o["k"] if c["kind"] != "dense" else m["k"] <= o["k"] for m, o in zip(got, info)), (got, info)
        for m, o in zip(got, info):
            if reached is None:  # the budget eps / sqrt(len(dim)) of the call
                assert abs(m["eps"] - o["eps"]) <= 1e-12 * o["eps"], (m["eps"], o["eps"])
            else:  # the device's own leftover over sqrt(N) (tn.round and Tensor(eps=) round every mode)
                assert abs(m["eps"] - calls["round_tucker"][-1]["eps"] / np.sqrt(len(info))) <= 1e-12 * m["eps"]
        if reached is not None or (c["kind"] == "dense" and "eps" in c):
            eps = c.get("eps", c.get("round", {}).get("eps"))
            d = calls["round_tucker"][-1]["dense"]
            r_dev = float(np.linalg.norm(d - dense)) / nrm
            want = (1 + eps) / (1 + r_dev) - 1
            assert abs(calls["round_tucker"][-1]["eps"] - want) <= 1e-7, (calls["round_tucker"][-1]["eps"], want)
    else:
        assert not calls["round_tucker"] or c["kind"] != "dense" and "round_tucker" in c
    # (a) ranks
    margins = []
    for m in (info or []):
        want, margin, nmargin = oracle_rank(m["sv"], dict(eps=m["eps"], rmax=m["rmax"]), min(m["I"], m["k"]), noise)
        margins.append((m["mu"], want, margin, nmargin))
    exact = all(a >= 1e-3 and b >= 1.0 for _, _, a, b in margins)
    tucker = [x.shape[1] for x in orc.cp_to_tt(list(dc))]
    otucker = [x.shape[1] for x in ocores]
    # per mode: whether its own decision has a margin, and the tail mass a mode without one may keep or drop
    # (relative to ||X||^2): the singular values between the smallest and the largest rank it could take
    mode_exact, slack2 = {}, 0.0
    for mu, want, a, b in margins:
        m = info[len(info) - 1 - mu]
        cap = min(m["rmax"] or 1 << 30, m["I"], m["k"])
        mode_exact[mu] = a >= 1e-3 and b >= 1.0
        if mode_exact[mu]:
            assert tucker[mu] == want, (mu, tucker, otucker)
            continue
        if m["eps"] > 1e-13:  # an eps rule at the noise: between its ranks at budgets moved by the noise
            # (the margin rule's own window: eps^2 moved by 1e-3 of itself and by 1e3 x noise)
            L = min(m["I"], m["k"])
            up = np.sqrt((m["eps"] * 1.001) ** 2 + 1e3 * noise)
            down = np.sqrt(max((m["eps"] * 0.999) ** 2 - 1e3 * noise, 0.0))
            lo = oracle_rank(m["sv"], dict(eps=up, rmax=m["rmax"]), L, noise)[0]
            hi = max(lo, oracle_rank(m["sv"], dict(eps=down, rmax=m["rmax"]), L, noise)[0])
        else:
            sv = m["sv"]
            lo, hi = min(int(np.sum(sv > (1e-10 if dtype == F64 else 1e-5) * sv[0])), cap), cap
        assert lo <= tucker[mu] <= hi, (mu, tucker, lo, hi)
        r0, r1 = min(lo, tucker[mu], otucker[mu]), max(hi, tucker[mu], otucker[mu])
        slack2 += float(np.sum(m["sv"][r0:r1] ** 2)) / nrm ** 2
    ranks_tt = t.ranks_tt.tolist()
    if exact:
        assert tucker == otucker and ranks_tt == [ocores[0].shape[0]] + [x.shape[2] for x in ocores], (tucker, ranks_tt)
        if dtype == F64:  # the reference's own ranks and error (CP: its Tucker ranks, see the module docstring)
            assert tucker == g[f"{name}/ranks_tucker"].tolist()
            if c["kind"] != "cp":
                assert ranks_tt == g[f"{name}/ranks_tt"].tolist()
                assert abs(e_dev - float(g[f"{name}/relerr"])) <= 1e-5, (e_dev, float(g[f"{name}/relerr"]))
    print(f"\n{name} {str(dtype)[6:]}: tucker {tucker} (oracle {otucker}) tt {ranks_tt} relerr {e_dev:.6g} "
          f"(oracle {e_orc:.6g}) margins {[(mu, f'{a:.2g}', f'{b:.2g}') for mu, _, a, b in margins]}")
    # (b) the error against the oracle's, beyond what the modes without a margin may move it: |e_dev^2 - e_orc^2| is at
    # most their slack, so |e_dev - e_orc| <= sqrt(slack2).  (c) the eps promise against the tensor decomposed (for a
    # 16- or 8-bit input, its values): relerr - eps with no allowance beyond the TOL entry
    print(f"  error slack of the modes without a margin: {np.sqrt(slack2):.3g}")
    bound("relerr", dtype, max(abs(e_dev - e_orc) - np.sqrt(slack2), 0.0))
    eps = eps_rule(c)
    if eps is not None:
        print(f"  eps promise: relerr {e_dev:.6g} eps {eps:.6g}")
        bound("eps_noise", dtype, max(e_dev - eps, 0.0))
    # (d) subspaces on gapped modes whose own decision has a margin and whose input did not depend on a rank decided at
    # the noise (every mode visited before it has the oracle's rank)
    for i, m in enumerate(info or []):
        mu, r = m["mu"], tucker[m["mu"]]
        sv = m["sv"]
        before_same = all(tucker[p["mu"]] == otucker[p["mu"]] for p in info[:i])
        if mode_exact[mu] and before_same and r < len(sv) and sv[r] < 0.5 * sv[r - 1] and sv[r - 1] > 1e-6 * sv[0]:
            bound("angle", dtype, principal_sin(dU[mu], oUs[mu]))
    ortho = [U for U in dU if U is not None]
    gauge = max([float(np.abs(U.T @ U - np.eye(U.shape[1])).max()) for U in ortho] + [0.0])
    if info is not None or c["kind"] != "dense" or "ranks_tt" in c:
        tt = orc.cp_to_tt(list(dc))
        gauge = max([gauge] + [float(np.abs(x.reshape(x.shape[0], -1) @ x.reshape(x.shape[0], -1).T - np.eye(x.shape[0])).max())
                               for x in tt[1:]])
    bound("gauge", dtype, gauge)
    # (f) tucker_core() and decompress_tucker_factors() against the oracle's contraction of the device's own cores
    core = widen(t.tucker_core())
    want = orc.tucker_core(dc)
    comp = float(np.abs(core - want).max() / max(np.abs(want).max(), 1e-300))
    dec = t.decompress_tucker_factors()
    full = orc.tucker_full(dc, dU)
    comp = max(comp, float(np.abs(orc.tucker_full([widen(x) for x in dec.cores], [None] * len(dc)) - full).max()
                           / np.abs(full).max()))
    bound("compose", dtype, comp)


@pytest.mark.gpu
def test_cp_on_tucker_core_is_a_composition():
    """Tensor(X, ranks_cp=R, ranks_tucker=S): the Tucker factors of Tensor(X, ranks_tucker=S), and ops.cp_als on its
    Tucker core from the same random start (tensor.py:278-302), bit for bit."""
    import tntorch_b200 as tnb
    from tntorch_b200 import ops

    rng = np.random.default_rng(9)
    fac = [rng.standard_normal((s, 3)) for s in (14, 12, 10)]
    X = torch.as_tensor(np.einsum("ar,br,cr->abc", *fac) + 1e-3 * rng.standard_normal((14, 12, 10))).cuda()
    for dtype in (F64, F32):
        Xd = X.to(dtype)
        tk = tnb.Tensor(Xd, ranks_tucker=4)
        torch.manual_seed(5)
        t = tnb.Tensor(Xd, ranks_cp=3, ranks_tucker=4, max_iter=7, tol=1e-12)
        assert all(torch.equal(a, b) for a, b in zip(t.Us, tk.Us))
        core = tk.tucker_core().contiguous()
        torch.manual_seed(5)
        init = [torch.randn(sh, 3, dtype=core.dtype, device="cuda") for sh in core.shape]
        want = ops.cp_als(core, 3, max_iter=7, tol=1e-12, init=init)
        assert all(torch.equal(a, b) for a, b in zip(t.cores, want))


def _abs_close(dev, orc_cores):
    worst = 0.0
    for a, b in zip(dev, orc_cores):
        if a is None:
            continue
        worst = max(worst, float(np.abs(np.abs(a) - np.abs(b)).max() / max(np.abs(b).max(), 1e-300)))
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("kind", ["tt", "cp", "tt_tucker"])
def test_orthogonalisation_against_oracle(kind, dtype):
    """left_/right_orthogonalize, orthogonalize(mu) for every mu and factor_orthogonalize on a batch of two: the tensor
    is unchanged, and every core and factor equals the oracle's QR result up to the signs of its rows and columns."""
    import tntorch_b200 as tnb

    shape, B = (6, 5, 7, 4), 2
    rng = np.random.default_rng({"tt": 1, "cp": 2, "tt_tucker": 3}[kind])
    samples = []
    for _ in range(B):
        if kind == "cp":
            cs, us = [rng.standard_normal((I, 3)) for I in shape], [None] * 4
        else:
            cs = cases.random_tt((4, 5, 3, 4) if kind == "tt_tucker" else shape, [3, 4, 3], int(rng.integers(1000)))
            us = [rng.standard_normal((I, c.shape[1])) for I, c in zip(shape, cs)] if kind == "tt_tucker" else [None] * 4
        samples.append((cs, us))

    def batch():
        cores = [torch.as_tensor(np.stack([s[0][n] for s in samples])).to(dtype).cuda() for n in range(4)]
        Us = None if kind != "tt_tucker" else [torch.as_tensor(np.stack([s[1][n] for s in samples])).to(dtype).cuda()
                                               for n in range(4)]
        return tnb.Tensor(cores, Us=Us, batch=True)

    def widened(t, b):
        return [widen(c[b]) for c in t.cores], [None if U is None else widen(U[b]) for U in t.Us]

    worst_q = worst_d = 0.0
    ops_list = [("orthogonalize", mu) for mu in range(4)] + [("left", mu) for mu in range(3)] + \
               [("right", mu) for mu in range(1, 4)] + [("factor", mu) for mu in range(4)]
    for op, mu in ops_list:
        t = batch()
        start = [widened(t, b) for b in range(B)]
        {"orthogonalize": t.orthogonalize, "left": t.left_orthogonalize, "right": t.right_orthogonalize,
         "factor": t.factor_orthogonalize}[op](mu)
        for b in range(B):
            cs, us = [x.copy() for x in start[b][0]], [None if U is None else U.copy() for U in start[b][1]]
            if op == "orthogonalize":
                orc.orthogonalize(cs, us, mu)
            elif op == "factor":
                orc.factor_orthogonalize(cs, us, mu)
            else:
                orc.cp_to_tt(cs)
                orc.factor_orthogonalize(cs, us, mu)
                (orc.left_orthogonalize if op == "left" else orc.right_orthogonalize)(cs, mu)
            dc, du = widened(t, b)
            assert [x.shape for x in orc.cp_to_tt(list(dc))] == [x.shape for x in orc.cp_to_tt(list(cs))], (op, mu)
            worst_q = max(worst_q, _abs_close(orc.cp_to_tt(list(dc)), orc.cp_to_tt(list(cs))), _abs_close(du, us))
            full0 = orc.tucker_full(*start[b])
            worst_d = max(worst_d, float(np.linalg.norm(orc.tucker_full(dc, du) - full0) / np.linalg.norm(full0)))
    print(f"\northogonalisation {kind} {str(dtype)[6:]}: cores {worst_q:.3g} tensor {worst_d:.3g}")
    bound("ortho", dtype, worst_q)
    bound("ortho_dense", dtype, worst_d)


@pytest.mark.gpu
def test_batched_tucker_is_refused():
    import tntorch_b200 as tnb

    X = torch.randn(2, 6, 5, 4, dtype=F64, device="cuda")
    with pytest.raises(NotImplementedError):
        tnb.Tensor(X, ranks_tucker=2, batch=True)
    t = tnb.Tensor(X, ranks_tt=3, batch=True)
    with pytest.raises(NotImplementedError):
        t.round_tucker(rmax=2)


@pytest.mark.gpu
def test_exact_tt_past_the_eigensolver_limit_is_refused():
    """Tensor(X, ranks_tucker=) starts from the exact TT; a 20^4 tensor's middle Gram is 400 x 400 of rank 400."""
    import tntorch_b200 as tnb

    X = torch.as_tensor(np.random.default_rng(0).standard_normal((20, 20, 20, 20))).cuda()
    with pytest.raises(NotImplementedError, match="240"):
        tnb.Tensor(X, ranks_tucker=3)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(REFUSED))
def test_refused_rounding_leaves_the_tensor_as_it_was(name):
    import tntorch_b200 as tnb

    r = REFUSED[name]
    t = tnb.Tensor([torch.as_tensor(x).cuda() for x in cases.make_tucker_input(r["spec"])[0]])
    cores, Us = list(t.cores), list(t.Us)
    saved = [x.clone() for x in cores]
    call = "round_tucker" if "round_tucker" in r else "round"
    with pytest.raises(NotImplementedError, match="240"):
        getattr(t, call)(**r[call])
    assert len(t.cores) == len(cores) and all(a is b for a, b in zip(t.cores, cores))
    assert all(torch.equal(a, b) for a, b in zip(t.cores, saved)) and t.Us == Us


# ---------------------------------------------------------------------------------------------- launched eigensolvers
# the direct solvers by their kernels; ChFSI and the adaptive solve by the random start of their subspace
# (random_fill_kernel, launched by nothing else on this path); their Rayleigh-Ritz steps may launch a Jacobi kernel
_DIRECT = {"jac2_f64": "jacobi2_eigh_kernel<double>", "jac2_mixed": "jacobi2_mixed_kernel",
           "onesided_smem": "jacobi_eigh_kernel", "onesided_gmem": "jacobi_eigh_kernel"}
_EIG_KERNEL = dict(_DIRECT, chfsi="random_fill_kernel", adaptive="random_fill_kernel")
PROFILED = [n for n, c in CASES.items() if c["kind"] == "tt" and "round_tucker" in c]


def trace_cases():
    """{name: [kernel names]} of one round_tucker per PROFILED case in fp64; run in a process of its own (late in a
    long process that has profiled before, the activity trace has come back without some of the kernels)."""
    import tntorch_b200 as tnb
    from torch.profiler import ProfilerActivity, profile

    out = {}
    for name in PROFILED:
        c = CASES[name]
        _, cores, Us = case_input(c, F64)
        t = tnb.Tensor(cores, Us=Us if Us[0] is not None else None)
        tnb.round_tucker(t, **c["round_tucker"])
        torch.cuda.synchronize()
        names = []
        for _ in range(3):
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                tnb.round_tucker(t, **c["round_tucker"])
                torch.cuda.synchronize()
            names = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
            if names:
                break
        out[name] = names
    return out


@pytest.fixture(scope="module")
def traced():
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here, os.environ.get("PYTHONPATH", "")]))
    code = "import json, test_gpu_tucker_paths as t; print('TRACE ' + json.dumps(t.trace_cases()))"
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=os.path.dirname(here),
                       timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    line = [x for x in r.stdout.splitlines() if x.startswith("TRACE ")][-1]
    return json.loads(line[len("TRACE "):])


@pytest.mark.gpu
@pytest.mark.parametrize("name", PROFILED)
def test_launched_eigensolvers_match_restatement(name, traced):
    """Every eigensolver the restatement names ran; with no subspace solve in the case, no other one did."""
    names = traced[name]
    assert names, "the profiler recorded no kernel"
    plan = mode_plan(CASES[name])
    want = {_EIG_KERNEL[p["eig"]] for p in plan if p["eig"] in _EIG_KERNEL}
    seen = {k for k in set(_EIG_KERNEL.values()) if any(k in n for n in names)}
    print(f"\n{name}: eigensolvers {[p['eig'] for p in plan]} launched {sorted(seen)}")
    assert want <= seen, (want, seen)
    if all(p["eig"] in _DIRECT for p in plan):
        assert seen == want, (want, seen)
