"""TT -> dense: the left-to-right chain of Tensor.torch() against the one-call path Tensor.torch(dtype=) (tnb_tt_decompress),
alternating in one process, CUDA-event timed.

    python scripts/bench_decompress.py --out DIR [--runs 3] [--steps 20] [--warmup 3]

Shapes: randn cores of 64^5 at TT-rank 32 (the cores `tn.Tensor(randn(64^5), ranks_tt=32)` has the shape of), 16^8 at
rank 32 and the 3-mode (256, 4096, 256) at rank 64.  Per shape and variant: ms per call (median and spread over the runs,
`steps` calls each), GB/s of result written and that rate as a fraction of the data-sheet 3.35 TB/s.  Variants: chain
(`t.torch()`), chain_to_bf16 (`t.torch().to(torch.bfloat16)`, what a 16-bit result costs through the chain), and the one
call to fp32, bf16 and fp16; a variant that does not fit in device memory is reported as such.  The card's name and power
limit are read in the same process.  Measurement only: writes DIR/bench_decompress.json.
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

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
SHAPES = {"64^5_r32": ([64] * 5, 32), "16^8_r32": ([16] * 8, 32), "256x4096x256_r64": ([256, 4096, 256], 64)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch

    import tntorch_b200 as tnb

    if not torch.cuda.is_available():
        raise SystemExit("bench_decompress: needs a CUDA device")
    out = {"card": card(), "hbm_datasheet_bytes_per_s": HBM_BYTES_PER_S, "runs": a.runs, "steps": a.steps}
    for name, (shape, r) in SHAPES.items():
        g = torch.Generator(device="cuda").manual_seed(108)
        rs = [1] + [r] * (len(shape) - 1) + [1]
        t = tnb.Tensor([torch.randn(rs[k], shape[k], rs[k + 1], generator=g, device="cuda") / math.sqrt(rs[k])
                        for k in range(len(shape))])
        numel = math.prod(shape)
        variants = {
            "chain": (lambda: t.torch(), 4),
            "chain_to_bf16": (lambda: t.torch().to(torch.bfloat16), 2),
            "one_call_fp32": (lambda: t.torch(dtype=torch.float32), 4),
            "one_call_bf16": (lambda: t.torch(dtype=torch.bfloat16), 2),
            "one_call_fp16": (lambda: t.torch(dtype=torch.float16), 2),
        }
        res = {"numel": numel}
        for k in list(variants):  # a variant that does not fit in memory is reported as such and left out
            try:
                for _ in range(a.warmup):
                    variants[k][0]()
                torch.cuda.synchronize()
            except torch.OutOfMemoryError:
                res[k] = "out of memory"
                del variants[k]
            torch.cuda.empty_cache()
        ms = {k: [] for k in variants}
        for _ in range(a.runs):
            for k, (fn, _) in variants.items():  # alternating
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.steps):
                    fn()
                e1.record()
                e1.synchronize()
                ms[k].append(e0.elapsed_time(e1) / a.steps)
        if "chain" in variants and numel <= 1 << 31:
            f32, old = t.torch(dtype=torch.float32), t.torch()
            res["one_call_vs_chain_rel_diff"] = float(torch.linalg.vector_norm(f32 - old) / torch.linalg.vector_norm(old))
            del f32, old
        for k, (_, esize) in variants.items():
            med = statistics.median(ms[k])
            gbs = numel * esize / (med * 1e-3) / 1e9
            res[k] = dict(ms=med, spread_ms=max(ms[k]) - min(ms[k]), runs_ms=ms[k], result_gb_s=gbs,
                          fraction_of_datasheet_hbm=gbs * 1e9 / HBM_BYTES_PER_S)
        out[name] = res
        del t
        torch.cuda.empty_cache()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_decompress.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
