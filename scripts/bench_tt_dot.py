"""Inner products of tensor trains: the one library call (ops.tt_dot / tt_dot_batch, tnb_tt_dot) against the einsum
chain the package ran before it (one fp64 torch.einsum per mode and pair), alternating in one process, CUDA-event timed.

    python scripts/bench_tt_dot.py --out DIR [--runs 3] [--steps 5] [--warmup 2]

Workloads (fp64): one config-3 pair (128^10, both rank 64); a batch of 64 config-3 squared norms; one rank-256 pair on
64^8 (ranks 64, 256 x 5, 64); and tn.relative_error(t, round_tt(t, rmax=16)) at config 3, whose three dots come from one
call (the rounding itself is done once, outside the timing).  The einsum arm is the yardstick only.

Per workload and arm: ms per call, median and spread over `runs` alternating runs of `steps` calls.  The flops are
those of the association order the library picks (2 n x its multiply-adds, per mode and pair).  They are set against
the fp64 mma.sync peak measured in the same process (ops.measure_f64_mma_peak): for the whole call, and, from a
torch.profiler run of its own, for the tensor-core kernels over the flops of the modes they run.  The card's name and
power limit are read in the same process.  Writes DIR/bench_tt_dot.json.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def flops(shape, ranks_a, ranks_b):
    """(all, on the tensor-core path) flops of one pair in the order ttd_order picks."""
    import ttd_model as tm

    tot = tc = 0
    for k, n in enumerate(shape):
        ra, rb, rao, rbo = ranks_a[k], ranks_b[k], ranks_a[k + 1], ranks_b[k + 1]
        f = 2 * n * min(rao * rb * (ra + rbo), rbo * ra * (rb + rao))
        tot += f
        swap = tm.order(ra, rb, rao, rbo)
        roles = (rb, ra, rbo, rao) if swap else (ra, rb, rao, rbo)
        tc += f if tm.mode_path(*roles) == tm.TC else 0
    return tot, tc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_tt_dot: needs a CUDA device")
    import tntorch_b200 as tnb
    from tntorch_b200 import ops

    os.makedirs(a.out, exist_ok=True)
    peak, _ = ops.measure_f64_mma_peak()
    res = {"card": card(), "mma_sync_f64_tflops_measured": peak, "workloads": {}}
    print(res["card"], f"mma.sync f64 {peak:.1f} TFLOP/s", flush=True)
    g = torch.Generator(device="cuda").manual_seed(0)

    def train(shape, ranks):
        r = [1] + ranks + [1]
        return [torch.randn(r[k], shape[k], r[k + 1], device="cuda", dtype=torch.float64, generator=g) / r[k] ** 0.5
                for k in range(len(shape))]

    def einsum_dot(x, y):
        m = torch.ones(1, 1, dtype=torch.float64, device="cuda")
        for p, q in zip(x, y):
            m = torch.einsum("ab,aic,bid->cd", m, p.double(), q.double())
        return m[0, 0]

    def ranks_of(cs):
        return [1] + [int(c.shape[2]) for c in cs]

    c3 = [128] * 10
    t64 = train(c3, [64] * 9)
    u64 = train(c3, [64] * 9)
    norms = [train(c3, [64] * 9) for _ in range(64)]
    s256 = [64] * 8
    a256, b256 = train(s256, [64] + [256] * 5 + [64]), train(s256, [64] + [256] * 5 + [64])
    t = tnb.Tensor(t64)
    r = tnb.round_tt(t, rmax=16)

    def relerr_einsum():
        aa, rr, ar = einsum_dot(t.cores, t.cores), einsum_dot(r.cores, r.cores), einsum_dot(t.cores, r.cores)
        return float(torch.sqrt((aa + rr - 2 * ar).clamp(0)) / torch.sqrt(aa.clamp(0)))

    work = {
        "cfg3_pair_r64": ([(t64, u64)], lambda: ops.tt_dot(t64, u64), lambda: einsum_dot(t64, u64)),
        "cfg3_64_norms_r64": ([(x, x) for x in norms], lambda: ops.tt_dot_batch([(x, x) for x in norms]),
                              lambda: torch.stack([einsum_dot(x, x) for x in norms])),
        "64^8_pair_r256": ([(a256, b256)], lambda: ops.tt_dot(a256, b256), lambda: einsum_dot(a256, b256)),
        "cfg3_relerr_round16": ([(t.cores, t.cores), (r.cores, r.cores), (t.cores, r.cores)],
                                lambda: tnb.relative_error(t, r), relerr_einsum),
    }
    from torch.profiler import ProfilerActivity, profile

    for name, (pairs, ours, ref) in work.items():
        arms = {"ours": ours, "einsum": ref}
        o, e = ours(), ref()
        o, e = torch.as_tensor(o, dtype=torch.float64).cpu(), torch.as_tensor(e, dtype=torch.float64).cpu()
        rel = float((o - e).abs().max() / e.abs().max())
        times = {k: [] for k in arms}
        for _ in range(a.runs):
            for k, f in arms.items():
                for _ in range(a.warmup):
                    f()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                for _ in range(a.steps):
                    f()
                e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1) / a.steps)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                ours()
            torch.cuda.synchronize()
        kern = {e.key: e.device_time_total / a.steps / 1e3 for e in prof.key_averages() if e.device_time_total > 0}
        fl = [flops([int(c.shape[1]) for c in x], ranks_of(x), ranks_of(y)) for x, y in pairs]
        tot, tc = sum(f[0] for f in fl), sum(f[1] for f in fl)
        tc_ms = sum(v for k, v in kern.items() if "ttd_mode_tc_kernel" in k)
        med = statistics.median(times["ours"])
        res["workloads"][name] = dict(
            pairs=len(pairs), ms={k: dict(median=statistics.median(v), min=min(v), max=max(v)) for k, v in times.items()},
            rel_diff_to_einsum=rel, gflop=tot / 1e9, gflop_tensor_core_modes=tc / 1e9,
            call_fraction_of_f64_mma_peak=tot / (med * 1e-3) / (peak * 1e12),
            tc_kernels_ms=tc_ms, tc_kernels_fraction_of_f64_mma_peak=(tc / (tc_ms * 1e-3) / (peak * 1e12)) if tc_ms else None,
            kernels_ms=kern)
        print(name, json.dumps({k: res["workloads"][name][k] for k in ("ms", "rel_diff_to_einsum", "gflop",
                                                                         "call_fraction_of_f64_mma_peak",
                                                                         "tc_kernels_fraction_of_f64_mma_peak")}),
              flush=True)
    with open(os.path.join(a.out, "bench_tt_dot.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
