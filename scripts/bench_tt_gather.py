"""Entries of tensor trains at many multi-indices: the one library call (ops.tt_gather, tnb_tt_gather) against the
torch bmm chain (cross._evaluate_tt_at, which forms core[:, idx, :] per mode) where it fits in memory, and against
ops.cross_tt_eval (fp64, ranks up to 64) where it applies; alternating in one process, CUDA-event timed.

    python scripts/bench_tt_gather.py --out DIR [--runs 3] [--steps 5] [--warmup 2]

Workloads: the config-3 train (128^10, rank 64, fp64) at P = 2^18 and 2^20; 64^5 at rank 32 in fp32 at P = 2^22; a
cross-validation size (32^6, rank 10, fp64, P = 1000); rank 256 on 16^8 in fp32 (P = 2^16).

Per workload and arm: ms per call, median and spread over `runs` alternating runs of `steps` calls.  The grouped path's
state traffic (the first mode writes P r, each inner mode reads and writes it, the last reads it; plus the indices) is
set against the data-sheet 3.35 TB/s, and the multiply-adds of the tensor-core modes, from a torch.profiler run of its
own, against the mma.sync peak measured in the same process (fp64 DMMA, or TF32 with the 3xTF32 split's three MMAs per
product).  The card's name and power limit are read in the same process.  Writes DIR/bench_tt_gather.json.
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
HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def traffic(shape, ranks, P, es):
    """Bytes of state the grouped path must move, and the indices it reads."""
    N = len(shape)
    b = P * N * 8 + P * ranks[1] * es
    for k in range(1, N):
        b += P * ranks[k] * es + P * ranks[k + 1] * es
    return b


def flops(shape, ranks, P):
    """(all, tensor-core modes) flops of the chain."""
    import ttg_model as tm

    tot = tc = 0
    for k in range(1, len(shape)):
        f = 2 * P * ranks[k] * ranks[k + 1]
        tot += f
        tc += f if tm.mode_path(ranks[k], ranks[k + 1]) == tm.TC else 0
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
        raise SystemExit("bench_tt_gather: needs a CUDA device")
    from tntorch_b200 import ops
    from tntorch_b200.cross import _evaluate_tt_at

    os.makedirs(a.out, exist_ok=True)
    f64_peak, _ = ops.measure_f64_mma_peak()
    tf32_peak, _ = ops.measure_tf32_peak()
    res = {"card": card(), "mma_sync_f64_tflops_measured": f64_peak, "mma_sync_tf32_tflops_measured": tf32_peak,
           "workloads": {}}
    print(res["card"], f"mma.sync f64 {f64_peak:.1f}, tf32 {tf32_peak:.1f} TFLOP/s", flush=True)
    g = torch.Generator(device="cuda").manual_seed(0)

    def train(shape, r, dt):
        r = [1] + [r] * (len(shape) - 1) + [1] if isinstance(r, int) else r
        return [(torch.randn(r[k], shape[k], r[k + 1], device="cuda", dtype=torch.float64, generator=g) / r[k] ** 0.5)
                .to(dt) for k in range(len(shape))], r

    def points(shape, P):
        return torch.stack([torch.randint(0, n, (P,), device="cuda", generator=g) for n in shape], dim=1)

    W = {
        "cfg3_r64_f64_P2^18": ([128] * 10, 64, torch.float64, 1 << 18),
        "cfg3_r64_f64_P2^20": ([128] * 10, 64, torch.float64, 1 << 20),
        "64^5_r32_f32_P2^22": ([64] * 5, 32, torch.float32, 1 << 22),
        "32^6_r10_f64_P1000": ([32] * 6, 10, torch.float64, 1000),
        "16^8_r256_f32_P2^16": ([16] * 8, [1, 16, 256, 256, 256, 256, 256, 16, 1], torch.float32, 1 << 16),
    }
    from torch.profiler import ProfilerActivity, profile

    for name, (shape, r, dt, P) in W.items():
        cores, ranks = train(shape, r, dt)
        idx = points(shape, P)
        cols = [idx[:, k].contiguous() for k in range(len(shape))]
        es = 8 if dt == torch.float64 else 4
        arms = {"tt_gather": lambda: ops.tt_gather(cores, idx, check=False)}
        free = torch.cuda.mem_get_info()[0]
        if 3 * P * max(ranks) ** 2 * es < free / 2:
            arms["bmm_chain"] = lambda: _evaluate_tt_at(cores, cols)
        else:
            print(name, "bmm chain skipped: its per-mode slices would not fit", flush=True)
        if dt == torch.float64 and max(ranks) <= 64:
            c4, i32 = [c[None] for c in cores], idx.int()
            arms["cross_tt_eval"] = lambda: ops.cross_tt_eval(c4, i32)[0]
        ours = arms["tt_gather"]()[0, :, 0]
        diffs = {k: float((f().reshape(-1) - ours).abs().max() / ours.abs().max()) for k, f in arms.items()
                 if k != "tt_gather"}
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
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                arms["tt_gather"]()
            torch.cuda.synchronize()
        kern = {e.key: e.device_time_total / a.steps / 1e3 for e in prof.key_averages() if e.device_time_total > 0}
        tot, tc = flops(shape, ranks, P)
        tc_ms = sum(v for k, v in kern.items() if "ttg_step_tc_kernel" in k)
        peak = f64_peak if dt == torch.float64 else tf32_peak / 3  # 3xTF32: three MMAs per product
        med = statistics.median(times["tt_gather"])
        bytes_ = traffic(shape, ranks, P, es)
        res["workloads"][name] = dict(
            P=P, ms={k: dict(median=statistics.median(v), min=min(v), max=max(v)) for k, v in times.items()},
            rel_diff_to_tt_gather=diffs, state_gb=bytes_ / 1e9, hbm_bound_ms=bytes_ / HBM * 1e3,
            call_fraction_of_hbm_bound=bytes_ / HBM * 1e3 / med, gflop=tot / 1e9, gflop_tensor_core_modes=tc / 1e9,
            tc_kernels_ms=tc_ms,
            tc_kernels_fraction_of_mma_peak=(tc / (tc_ms * 1e-3) / (peak * 1e12)) if tc_ms else None,
            kernels_ms=kern)
        print(name, json.dumps({k: res["workloads"][name][k] for k in ("ms", "rel_diff_to_tt_gather", "hbm_bound_ms",
                                                                         "call_fraction_of_hbm_bound",
                                                                         "tc_kernels_fraction_of_mma_peak")}),
              flush=True)
        del cores, idx, cols, arms
        torch.cuda.empty_cache()
    with open(os.path.join(a.out, "bench_tt_gather.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
