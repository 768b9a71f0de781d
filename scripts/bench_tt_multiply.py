"""Y = X M for a TT-matrix M: the one library call (tn.tt_multiply, tnb_tt_multiply) against the reference's einsum chain
restated in torch and against the dense product X @ M, alternating in one process, CUDA-event timed.

    python scripts/bench_tt_multiply.py --out DIR [--runs 3] [--steps 10] [--warmup 3]

Workloads (batch, input dims, output dims, rank): 8192 x (8^4 -> 8^4) at ranks 16 and 32, 65536 x (4^5 -> 4^5) at rank 8,
and the reference test's 30 x ([11, 3] -> [23, 2]) at rank 50 (a latency case).  Arms: `ours`; `einsum`, the reference's
chain (X.T, one torch.einsum per core) in fp32 with TF32 matmuls off; `dense`, X @ ttm.torch(dtype=torch.float32) by
torch.matmul with TF32 off (M formed once, outside the timing).  The torch arms are yardsticks only.

Per workload and arm: ms per call, median and spread over `runs` alternating runs of `steps` calls.  A separate
torch.profiler run gives each kernel of our call its time; each step is set against its bound: the algorithmic bytes
4 (M K + M N) at 3.35 TB/s (H100 SXM data sheet) or the flops 2 M K N at one third of the measured TF32 rate of the MMA
the step issues (mma.sync on the tensor-core path, measured here with ops.measure_tf32_peak; 3xTF32 issues three), the
larger of the two.  The card's name and power limit are read in the same process.  Writes DIR/bench_tt_multiply.json.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
WORKLOADS = {
    "8^4_r16": (8192, [8] * 4, [8] * 4, 16),
    "8^4_r32": (8192, [8] * 4, [8] * 4, 32),
    "4^5_r8": (65536, [4] * 5, [4] * 5, 8),
    "ref_30x33_r50": (30, [11, 3], [23, 2], 50),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def step_counts(nb, idims, odims, ranks):
    """(M, K, N, bytes, flops) of each step, fp32"""
    out = []
    for k in range(len(idims)):
        M = nb * math.prod(idims[k + 1:]) * math.prod(odims[:k])
        K, N = idims[k] * ranks[k], odims[k] * ranks[k + 1]
        out.append((M, K, N, 4 * (M * K + M * N), 2 * M * K * N))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_tt_multiply: needs a CUDA device")
    import tntorch_b200 as tnb
    from tntorch_b200 import ops
    from tntorch_b200.callers import _tt_multiply_einsum
    import ttm_model as tm

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    os.makedirs(a.out, exist_ok=True)
    mma_tf32, _ = ops.measure_tf32_peak()
    res = {"card": card(), "mma_sync_tf32_tflops_measured": mma_tf32, "workloads": {}}
    print(res["card"], f"mma.sync tf32 {mma_tf32:.1f} TFLOP/s", flush=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, (nb, idims, odims, r) in WORKLOADS.items():
        d = len(idims)
        ranks = [1] + [r] * (d - 1) + [1]
        cores = [torch.randn(ranks[k], idims[k], odims[k], ranks[k + 1], device="cuda", generator=g) /
                 math.sqrt(ranks[k] * idims[k]) for k in range(d)]
        ttm = tnb.TTMatrix(cores, ranks=ranks[1:-1], input_dims=idims, output_dims=odims)
        X = torch.randn(nb, math.prod(idims), device="cuda", generator=g)
        M = ttm.torch(dtype=torch.float32)
        arms = {"ours": lambda: tnb.tt_multiply(ttm, X), "einsum": lambda: _tt_multiply_einsum(ttm, X),
                "dense": lambda: torch.matmul(X, M)}
        Y = arms["ours"]()
        errs = {k: float(torch.linalg.norm(f() - arms["dense"]()) / torch.linalg.norm(arms["dense"]())) for k, f in arms.items()}
        del Y
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
        # per-step kernel times of our call, in a run of its own
        from torch.profiler import ProfilerActivity, profile

        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                arms["ours"]()
            torch.cuda.synchronize()
        kern = [(e.key, e.device_time_total / a.steps / 1e3) for e in prof.key_averages() if e.device_time_total > 0]
        evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "ttm_" in e.name),
                     key=lambda e: e.time_range.start)
        steps = step_counts(nb, idims, odims, ranks)
        paths = tm.paths(True, idims, odims, ranks, nb)
        per_call = tm.launches(True, idims, odims, ranks, nb)
        first = per_call - d  # the image launch precedes the steps
        rows = []
        for k, ((Mr, K, N, by, fl), p) in enumerate(zip(steps, paths)):
            kms = [evs[c * per_call + first + k].time_range.elapsed_us() / 1e3 for c in range(len(evs) // per_call)]
            t_hbm = by / HBM_BYTES_PER_S * 1e3
            t_mma = fl / (mma_tf32 / 3 * 1e12) * 1e3 if p == tm.TC else None
            bound, t_bound = ("HBM", t_hbm) if t_mma is None or t_hbm >= t_mma else ("3xTF32 mma.sync", t_mma)
            ms = statistics.median(kms) if kms else None
            rows.append(dict(step=k, M=Mr, K=K, N=N, bytes=by, flops=fl, path=tm.BRANCHES[p],
                             kernel=evs[first + k].name if len(evs) >= per_call else None, kernel_ms=ms, bound=bound,
                             bound_ms=t_bound, fraction_of_bound=(t_bound / ms) if ms else None))
        res["workloads"][name] = dict(
            batch=nb, input_dims=idims, output_dims=odims, rank=r,
            ms={k: dict(median=statistics.median(v), min=min(v), max=max(v)) for k, v in times.items()},
            rel_diff_to_dense=errs, kernels_ms=dict(kern), steps=rows,
            traffic_GB=sum(s[3] for s in steps) / 1e9, flops_T=sum(s[4] for s in steps) / 1e12,
            dense_flops_T=2 * nb * math.prod(idims) * math.prod(odims) / 1e12)
        print(name, json.dumps(res["workloads"][name]["ms"]), flush=True)
        for r_ in rows:
            print("   ", r_, flush=True)
        print("    kernels", kern, flush=True)
        del X, M, cores, ttm
        torch.cuda.empty_cache()
    with open(os.path.join(a.out, "bench_tt_multiply.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
