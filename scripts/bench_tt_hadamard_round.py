"""Rounding the elementwise product of two tensor trains: the one library call (ops.tt_hadamard_round,
tnb_tt_hadamard_round) against the paths that existed before it, alternating in one process, CUDA-event timed.

    python scripts/bench_tt_hadamard_round.py --out DIR [--runs 3] [--steps 2] [--warmup 1] [--quick]

Workloads:
  c3sq     config 3 (128^10, rank 64, fp64) squared, rmax=16;
  64x5     [64]^5 fp32 at rank 32 x 32 (R = 1024), rmax=32, beside the reference on the host cores (when staged);
  32x8     [32]^8 fp64 at rank 16 x 16 (R = 256), rmax=64, against today's Kronecker cores + tt_round;
  reduce4  tn.reduce of four config-3 trains with operator.mul, rmax=16.
Every workload also runs a torch fp64 einsum restatement of the same Gram algorithm (cuBLAS), the on-GPU baseline.

Per workload and arm: ms per call, median and spread over `runs` alternating runs of `steps` calls.  The flops of the
left-Gram recurrence come from the shapes (2 I (ra^2 ra' rb^2 + ra ra'^2 rb^2 + ra'^2 rb^2 rb' + ra'^2 rb rb'^2) per
mode); a torch.profiler run of its own gives the time of the tensor-core GEMM kernels, set against the fp64 mma.sync peak
measured in the same process (ops.measure_f64_mma_peak).  The card's name and power limit are read in the same
process.  Writes DIR/bench_tt_hadamard_round.json.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def gl_flops(shape, ra, rb):
    f = 0
    for k in range(len(shape) - 1):
        a, b, ao, bo, I = ra[k], rb[k], ra[k + 1], rb[k + 1], shape[k]
        f += 2 * I * (a * a * ao * b * b + a * ao * ao * b * b + ao * ao * b * b * bo + ao * ao * b * bo * bo)
    return f


def einsum_gram_round(a, b, rmax):
    """The same Gram algorithm in torch fp64 einsums (cuBLAS): left Grams, then per bond Y, H, eigh, rank = rmax."""
    import torch

    N = len(a)
    a = [c.double() for c in a]
    b = [c.double() for c in b]
    GL = [torch.ones(1, 1, dtype=torch.float64, device=a[0].device)]
    for k in range(N - 1):
        ra, I, rao = a[k].shape
        rb, _, rbo = b[k].shape
        G = GL[k].reshape(ra, rb, ra, rb)
        out = torch.zeros(rao, rbo, rao, rbo, dtype=torch.float64, device=G.device)
        for i in range(I):
            T = torch.einsum("abcd,ax->bcdx", G, a[k][:, i])
            T = torch.einsum("bcdx,by->cdxy", T, b[k][:, i])
            T = torch.einsum("cdxy,cz->dxyz", T, a[k][:, i])
            out += torch.einsum("dxyz,dw->xyzw", T, b[k][:, i])
        GL.append(out.reshape(rao * rbo, rao * rbo))
    W = torch.ones(1, 1, dtype=torch.float64, device=a[0].device)
    for mu in range(N - 1, 0, -1):
        ra, I, rao = a[mu].shape
        rb, _, rbo = b[mu].shape
        rn = W.shape[1]
        Z = torch.einsum("xyj,biy->ixjb", W.reshape(rao, rbo, rn), b[mu])
        Y = torch.einsum("aix,ixjb->abij", a[mu], Z).reshape(ra * rb, I * rn)
        H = Y.T @ (GL[mu] @ Y)
        w, V = torch.linalg.eigh(0.5 * (H + H.T))
        V = V[:, -min(rmax, V.shape[1]):]
        W = Y @ V
    return W


def timed(fn, steps, warmup):
    import torch

    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--quick", action="store_true", help="skip the reference on the host and the einsum arm at config 3")
    a = ap.parse_args()
    import operator

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_tt_hadamard_round: needs a CUDA device")
    import tntorch_b200 as tnb
    from tntorch_b200 import ops

    def tt(seed, shape, r, dtype, scale=1.0):
        g = torch.Generator().manual_seed(seed)
        rr = [1] + [r] * (len(shape) - 1) + [1]
        return [(scale * torch.randn(rr[k], shape[k], rr[k + 1], generator=g, dtype=torch.float64)).to(dtype).cuda()
                for k in range(len(shape))]

    peak, _ = ops.measure_f64_mma_peak()
    res = dict(card=card(), f64_mma_peak_tflops=peak, workloads={})
    c3 = tt(1, [128] * 10, 64, torch.float64, 1 / 8)
    W = {
        "c3sq": dict(arms={"fused": lambda: ops.tt_hadamard_round(c3, c3, rmax=16)},
                     flops=gl_flops([128] * 10, [1] + [64] * 9 + [1], [1] + [64] * 9 + [1])),
    }
    x5, y5 = tt(2, [64] * 5, 32, torch.float32), tt(3, [64] * 5, 32, torch.float32)
    W["64x5"] = dict(arms={"fused": lambda: ops.tt_hadamard_round(x5, y5, rmax=32),
                           "einsum": lambda: einsum_gram_round(x5, y5, 32)},
                     flops=gl_flops([64] * 5, [1] + [32] * 4 + [1], [1] + [32] * 4 + [1]))
    x8, y8 = tt(4, [32] * 8, 16, torch.float64), tt(5, [32] * 8, 16, torch.float64)
    W["32x8"] = dict(arms={"fused": lambda: ops.tt_hadamard_round(x8, y8, rmax=64),
                           "kronecker": lambda: ops.tt_round(ops.tt_hadamard(x8, y8), rmax=64),
                           "einsum": lambda: einsum_gram_round(x8, y8, 64)},
                     flops=gl_flops([32] * 8, [1] + [16] * 7 + [1], [1] + [16] * 7 + [1]))
    ts4 = [tnb.Tensor(tt(10 + k, [128] * 10, 64, torch.float64, 1 / 8)) for k in range(4)]
    W["reduce4"] = dict(arms={"fused": lambda: tnb.reduce(ts4, operator.mul, rmax=16)}, flops=None)
    if not a.quick:
        W["c3sq"]["arms"]["einsum"] = lambda: einsum_gram_round(c3, c3, 16)
    for name, w in W.items():
        times = {k: [] for k in w["arms"]}
        for _ in range(a.runs):
            for arm, fn in w["arms"].items():
                times[arm].append(timed(fn, a.steps, a.warmup))
        out = {arm: dict(ms_median=statistics.median(v), ms_min=min(v), ms_max=max(v)) for arm, v in times.items()}
        if w["flops"]:
            out["gl_tflop"] = w["flops"] / 1e12
        res["workloads"][name] = out
        print(name, json.dumps(out), flush=True)
    # kernel time of the tensor-core GEMMs at config 3 squared, from a profiler run of its own
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ops.tt_hadamard_round(c3, c3, rmax=16)
        torch.cuda.synchronize()
    tc_us = sum(e.device_time_total for e in prof.key_averages() if "tthr_gemm_tc_kernel" in e.key)
    all_us = sum(e.device_time_total for e in prof.key_averages())
    res["c3sq_kernels"] = dict(tc_gemm_ms=tc_us / 1e3, all_kernels_ms=all_us / 1e3,
                               gl_fraction_of_peak=W["c3sq"]["flops"] / (tc_us * 1e-6) / 1e12 / peak if tc_us else None)
    print("c3sq kernels", json.dumps(res["c3sq_kernels"]), flush=True)
    if not a.quick:
        from oracle import stage_ref

        ref = stage_ref.load()
        if ref is not None:
            xa = ref.Tensor([c.cpu() for c in x5])
            ya = ref.Tensor([c.cpu() for c in y5])
            t0 = time.perf_counter()
            try:
                ref.round_tt(xa * ya, rmax=32)
                res["workloads"]["64x5"]["reference_host_ms"] = (time.perf_counter() - t0) * 1e3
            except Exception as e:  # the reference's own limits (memory on the host)
                res["workloads"]["64x5"]["reference_host"] = f"{type(e).__name__}: {e}"[:200]
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_tt_hadamard_round.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
