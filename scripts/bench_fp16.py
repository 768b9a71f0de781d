"""fp16 against fp32 input on the flagship workload: randn(64^5) rounded to fp16, decomposed at TT-rank 32 as fp16 and
as the same values upcast to fp32, alternating in one process.

    python scripts/bench_fp16.py --out DIR [--runs 3] [--steps 5] [--warmup 3] [--batch 4] [--noise-only]

Per input type: one-call GElements/s (median and spread over the runs, `steps` timed calls each), batch GElements/s
(TTSVDBatchPlan over `batch` tensors), the step-0 Gram and projection ms from TNB_FLAG_PROFILE, and the relative error
against the fp16 data.  The card's name and power limit are read in the same process.  Also the noise of the fp16 and
the TF32 tensor-core Gram against the fp64 Gram of the same fp16 values: ||G_tc - (1 - c) G_fp64||_2 / ||G_fp64||_2, c
the least-squares shrink, on the inputs scripts/bench_bf16.py uses: randn(2^24, 64), randn(262144, 2048) and a rank-6
signal plus 1e-3 noise of 2^24 x 64.  Writes DIR/bench_fp16.json (DIR/bench_fp16_noise.json with --noise-only).
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


def gram_noise():
    import torch

    from tntorch_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(11)
    mats = {"randn_16777216x64": lambda: torch.randn(1 << 24, 64, generator=g, device="cuda"),
            "randn_262144x2048": lambda: torch.randn(262144, 2048, generator=g, device="cuda"),
            "rank6_noise1e-3_16777216x64": lambda: (torch.randn(1 << 24, 6, generator=g, device="cuda")
                                                    @ torch.randn(6, 64, generator=g, device="cuda")
                                                    + 1e-3 * torch.randn(1 << 24, 64, generator=g, device="cuda"))}
    out = {}
    for name, make in mats.items():
        A = make().to(torch.float16)
        n = A.shape[1]
        ref = torch.zeros(n, n, dtype=torch.float64, device="cuda")
        for i in range(0, A.shape[0], 1 << 20):
            B = A[i: i + (1 << 20)].double()
            ref += B.T @ B
        for kind, G in (("fp16", ops.gram_f16(A)), ("tf32", ops.gram(A.float(), tensorcore=True))):
            c = 1.0 - float((G * ref).sum() / (ref * ref).sum())
            nr = float(torch.linalg.matrix_norm(ref, ord=2))
            out[f"{name}/{kind}"] = dict(bias_c=c, noise_rel_2norm=float(torch.linalg.matrix_norm(G - (1 - c) * ref, ord=2)) / nr,
                                         raw_rel_2norm=float(torch.linalg.matrix_norm(G - ref, ord=2)) / nr)
        del A, ref
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--noise-only", action="store_true")
    a = ap.parse_args()
    import torch

    from tntorch_b200 import ops

    noise = gram_noise()
    if a.noise_only:
        out = {"card": card(), "gram_noise": noise}
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_fp16_noise.json"), "w") as f:
            json.dump(out, f, indent=1)
        print(json.dumps(out))
        return

    shape, r = [64] * 5, 32
    numel = 64 ** 5
    g = torch.Generator(device="cuda").manual_seed(108)
    Xh = torch.randn(shape, generator=g, device="cuda").to(torch.float16)
    inputs = {"fp16": Xh, "fp32": Xh.float()}
    plans = {k: ops.TTSVDPlan(shape, x.dtype, rmax=r) for k, x in inputs.items()}
    prof = {k: ops.TTSVDPlan(shape, x.dtype, rmax=r, profile=True) for k, x in inputs.items()}
    bplans = {k: ops.TTSVDBatchPlan(shape, x.dtype, a.batch, rmax=r) for k, x in inputs.items()}
    batches = {k: [x] * a.batch for k, x in inputs.items()}
    res = {k: dict(call=[], batch=[]) for k in inputs}
    for k in inputs:
        for _ in range(a.warmup):
            plans[k].run(inputs[k])
            bplans[k].run(batches[k])
    torch.cuda.synchronize()
    for _ in range(a.runs):
        for k in inputs:  # alternating
            t0 = time.perf_counter()
            for _ in range(a.steps):
                plans[k].run(inputs[k])
            torch.cuda.synchronize()
            res[k]["call"].append(a.steps * numel / (time.perf_counter() - t0) / 1e9)
            t0 = time.perf_counter()
            bplans[k].run(batches[k])
            torch.cuda.synchronize()
            res[k]["batch"].append(a.batch * numel / (time.perf_counter() - t0) / 1e9)
    out = {"card": card(), "shape": shape, "rank": r, "gram_noise": noise}
    for k in inputs:
        cores = plans[k].run(inputs[k])
        prof[k].run(inputs[k])
        info = prof[k].info
        out[k] = dict(
            call_gelem_s=dict(median=statistics.median(res[k]["call"]), spread=max(res[k]["call"]) - min(res[k]["call"]),
                              runs=res[k]["call"]),
            batch_gelem_s=dict(median=statistics.median(res[k]["batch"]),
                               spread=max(res[k]["batch"]) - min(res[k]["batch"]), runs=res[k]["batch"]),
            step0_gram_ms=info[8], step0_factor_ms=info[10], call_ms_profiled=info[4] + info[5] + info[6],
            speculative=int(plans[k].info[26]), kblocked_steps=int(plans[k].info[28]),
            rel_error_vs_fp16=ops.tt_relative_error(Xh, [c.clone() for c in cores]))
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_fp16.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
