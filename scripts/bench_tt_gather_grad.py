"""Forward plus backward of entries of tensor trains under autograd: the library (ops.tt_gather, whose backward is one
tnb_tt_gather_grad call) against the torch chain of core[:, idx, :] products under autograd where it fits in memory;
alternating in one process, CUDA-event timed.

    python scripts/bench_tt_gather_grad.py --out DIR [--runs 3] [--steps 3] [--warmup 1]

Workloads: the config-3 train (128^10, rank 64, fp64) at P = 2^18 and 2^20; 64^5 rank 32 fp32 at P = 2^22; [2]*20 rank
16 fp64 at P = 2^18 (two long buckets per mode: the chunked reduction); 32^6 rank 10 fp64 at P = 2^16 (below the
tensor-core envelope).

Per workload and arm: ms per forward + backward, median and spread over `runs` alternating runs of `steps` calls; the
library's forward alone, and its backward-to-forward ratio.  The backward's state traffic (bytes_model: the forward
recompute writes and reads each kept L_k; per mode the reduction reads L_k and W_k, the reverse step reads W_k and writes
W_{k-1}; plus the indices and the orders) is set against the data-sheet 3.35 TB/s.  The multiply-adds of the ttgg_ and
reverse-step kernels on the tensor cores, from a torch.profiler run of its own, are set against the mma.sync peaks
measured in the same process (fp64 DMMA, or TF32 with the 3xTF32 split's three MMAs per product).  The card's name and
power limit are read in the same process.  Writes DIR/bench_tt_gather_grad.json.
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


def bytes_model(shape, ranks, P, es):
    """Bytes the backward must move: indices and per-mode orders, the recomputed L_k written once and read by the next
    step and the reduction, W_k read by the reduction and the reverse step and written once."""
    N = len(shape)
    b = P * N * 8 + P * N * 4 * 4  # key, narrowed indices, counts, orders
    for k in range(1, N):
        b += 3 * P * ranks[k] * es  # L_k: written, read by the next step (k < N - 1) or not, read by the reduction
    for k in range(N):
        b += 2 * P * ranks[k + 1] * es + (P * ranks[k] * es if k > 0 else 0)  # W_k read twice, W_{k-1} written
    return b


def flops(shape, ranks, P):
    """(all, tensor-core) flops of the backward's recompute, reductions and reverse steps."""
    import ttg_model as tm

    tot = tc = 0
    for k in range(len(shape)):
        on_tc = tm.mode_path(ranks[k], ranks[k + 1]) == tm.TC
        f = 2 * P * ranks[k] * ranks[k + 1] * ((1 if k == 0 else 2) + (1 if 0 < k < len(shape) - 1 else 0))
        tot += f
        tc += f if on_tc else 0
    return tot, tc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_tt_gather_grad: needs a CUDA device")
    from tntorch_b200 import ops

    os.makedirs(a.out, exist_ok=True)
    f64_peak, _ = ops.measure_f64_mma_peak()
    tf32_peak, _ = ops.measure_tf32_peak()
    res = {"card": card(), "mma_sync_f64_tflops_measured": f64_peak, "mma_sync_tf32_tflops_measured": tf32_peak,
           "workloads": {}}
    print(res["card"], f"mma.sync f64 {f64_peak:.1f}, tf32 {tf32_peak:.1f} TFLOP/s", flush=True)
    g = torch.Generator(device="cuda").manual_seed(0)

    def train(shape, r, dt):
        r = [1] + [r] * (len(shape) - 1) + [1]
        return [(torch.randn(r[k], shape[k], r[k + 1], device="cuda", dtype=torch.float64, generator=g) / r[k] ** 0.5)
                .to(dt).requires_grad_() for k in range(len(shape))], r

    def points(shape, P):
        return torch.stack([torch.randint(0, n, (P,), device="cuda", generator=g) for n in shape], dim=1)

    def chain(cores, idx):
        s = cores[0][:, idx[:, 0], :]
        for k in range(1, len(cores)):
            s = torch.einsum("iaj,jak->iak", s, cores[k][:, idx[:, k], :])
        return s

    W = {
        "cfg3_r64_f64_P2^18": ([128] * 10, 64, torch.float64, 1 << 18),
        "cfg3_r64_f64_P2^20": ([128] * 10, 64, torch.float64, 1 << 20),
        "64^5_r32_f32_P2^22": ([64] * 5, 32, torch.float32, 1 << 22),
        "2^20_r16_f64_P2^18": ([2] * 20, 16, torch.float64, 1 << 18),
        "32^6_r10_f64_P2^16": ([32] * 6, 10, torch.float64, 1 << 16),
    }
    from torch.profiler import ProfilerActivity, profile

    for name, (shape, r, dt, P) in W.items():
        cores, ranks = train(shape, r, dt)
        idx = points(shape, P)
        w = torch.randn(1, P, 1, device="cuda", dtype=dt, generator=g)
        es = 8 if dt == torch.float64 else 4

        def lib_fb():
            for c in cores:
                c.grad = None
            (ops.tt_gather(cores, idx, check=False) * w).sum().backward()

        def lib_f():
            with torch.no_grad():
                ops.tt_gather(cores, idx, check=False)

        def chain_fb():
            for c in cores:
                c.grad = None
            (chain(cores, idx) * w).sum().backward()

        arms = {"tt_gather_grad": lib_fb, "tt_gather_forward": lib_f}
        free = torch.cuda.mem_get_info()[0]
        if 2 * len(shape) * P * max(ranks) ** 2 * es < free / 2:
            arms["torch_chain"] = chain_fb
        else:
            print(name, "torch chain skipped: its per-mode slices would not fit", flush=True)
        lib_fb()
        ours = [c.grad.clone() for c in cores]
        diffs = None
        if "torch_chain" in arms:
            chain_fb()
            diffs = max(float((c.grad - o).abs().max() / o.abs().max().clamp_min(1e-300)) for c, o in zip(cores, ours))
        del ours
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
                lib_fb()
            torch.cuda.synchronize()
        kern = {e.key: e.device_time_total / a.steps / 1e3 for e in prof.key_averages() if e.device_time_total > 0}
        tot, tc = flops(shape, ranks, P)
        tc_ms = sum(v for k, v in kern.items()
                    if "ttgg_reduce_tc_kernel" in k or ("ttg_step_tc_kernel" in k and "true" in k))
        bwd_ms = sum(v for k, v in kern.items() if "ttgg_" in k or ("ttg_" in k and "true" in k)
                     or "ttg_init_kernel" in k)
        peak = f64_peak if dt == torch.float64 else tf32_peak / 3
        fb = statistics.median(times["tt_gather_grad"])
        fwd = statistics.median(times["tt_gather_forward"])
        bytes_ = bytes_model(shape, ranks, P, es)
        res["workloads"][name] = dict(
            P=P, ms={k: dict(median=statistics.median(v), min=min(v), max=max(v)) for k, v in times.items()},
            backward_ms=fb - fwd, backward_to_forward=(fb - fwd) / fwd, rel_diff_chain_grads=diffs,
            backward_gb=bytes_ / 1e9, hbm_bound_ms=bytes_ / HBM * 1e3,
            backward_fraction_of_hbm_bound=bytes_ / HBM * 1e3 / (fb - fwd), gflop=tot / 1e9,
            gflop_tensor_core=tc / 1e9, backward_kernels_ms=bwd_ms, tc_kernels_ms=tc_ms,
            tc_kernels_fraction_of_mma_peak=(tc / (tc_ms * 1e-3) / (peak * 1e12)) if tc_ms else None,
            kernels_ms=kern)
        print(name, json.dumps({k: res["workloads"][name][k] for k in (
            "ms", "backward_ms", "backward_to_forward", "rel_diff_chain_grads", "hbm_bound_ms",
            "backward_fraction_of_hbm_bound", "tc_kernels_fraction_of_mma_peak")}), flush=True)
        del cores, idx, arms
        torch.cuda.empty_cache()
    with open(os.path.join(a.out, "bench_tt_gather_grad.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
