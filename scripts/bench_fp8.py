"""fp8 against fp16 and fp32 input on the flagship workload: randn(64^5) rounded to each fp8 format (e4m3fn, e5m2),
decomposed at TT-rank 32 as fp8 and as the same values upcast to fp16 and to fp32, alternating in one process.

    python scripts/bench_fp8.py --out DIR [--runs 3] [--steps 5] [--warmup 3] [--batch 4] [--noise-only]

Per format and input type: one-call GElements/s (median and spread over the runs, `steps` timed calls each), batch
GElements/s (TTSVDBatchPlan over `batch` tensors), the step-0 Gram and projection ms from TNB_FLAG_PROFILE with the bytes
and executed flops of those two kernels (computed from the shapes) and the rates they imply, and the relative error
against the fp8 data.  The card's name and power limit are read in the same process.  Also the noise of the fp8
tensor-core Gram against the fp64 Gram of the same fp8 values: ||G_f8 - (1 - c) G_fp64||_2 / ||G_fp64||_2, c the
least-squares shrink, on the inputs scripts/bench_bf16.py uses, rounded to each format: randn(2^24, 64),
randn(262144, 2048) and a rank-6 signal plus 1e-3 noise of 2^24 x 64.  Writes DIR/bench_fp8.json
(DIR/bench_fp8_noise.json with --noise-only).
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


def formats():
    import torch

    return {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}


def gram_noise():
    import torch

    from tntorch_b200 import ops

    out = {}
    for fname, dt in formats().items():
        g = torch.Generator(device="cuda").manual_seed(11)
        mats = {"randn_16777216x64": lambda: torch.randn(1 << 24, 64, generator=g, device="cuda"),
                "randn_262144x2048": lambda: torch.randn(262144, 2048, generator=g, device="cuda"),
                "rank6_noise1e-3_16777216x64": lambda: (torch.randn(1 << 24, 6, generator=g, device="cuda")
                                                        @ torch.randn(6, 64, generator=g, device="cuda")
                                                        + 1e-3 * torch.randn(1 << 24, 64, generator=g, device="cuda"))}
        for name, make in mats.items():
            A = make().to(dt)
            n = A.shape[1]
            ref = torch.zeros(n, n, dtype=torch.float64, device="cuda")
            for i in range(0, A.shape[0], 1 << 20):
                B = A[i: i + (1 << 20)].double()
                ref += B.T @ B
            G = ops.gram_f8(A)
            c = 1.0 - float((G * ref).sum() / (ref * ref).sum())
            nr = float(torch.linalg.matrix_norm(ref, ord=2))
            out[f"{name}/{fname}"] = dict(
                bias_c=c, noise_rel_2norm=float(torch.linalg.matrix_norm(G - (1 - c) * ref, ord=2)) / nr,
                raw_rel_2norm=float(torch.linalg.matrix_norm(G - ref, ord=2)) / nr)
            del A, ref
    return out


def step0_model(esize, rows=64 ** 4, n=64, r=32, vterms=2):
    """Bytes and executed flops of the step-0 kernels of 64^5 at rank r: the Gram reads the input once and computes one
    folded 128 x 128 tile over rows / 2 rows (fp8: only its two diagonal 64 x 64 blocks); the projection reads the input
    and writes the fp32 carry, and issues vterms products of the input with V (npad = r columns)."""
    gram_bytes = rows * n * esize
    gram_flops = 2 * (rows * n // 128) * 128 * (64 if esize == 1 else 128)
    proj_bytes = rows * n * esize + rows * r * 4
    proj_flops = 2 * rows * n * r * vterms
    return gram_bytes, gram_flops, proj_bytes, proj_flops


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

    os.makedirs(a.out, exist_ok=True)
    if a.noise_only:
        out = {"card": card(), "gram_noise": gram_noise()}
        with open(os.path.join(a.out, "bench_fp8_noise.json"), "w") as f:
            json.dump(out, f, indent=1)
        print(json.dumps(out))
        return

    shape, r = [64] * 5, 32
    numel = 64 ** 5
    out = {"card": card(), "shape": shape, "rank": r}
    for fname, dt in formats().items():
        g = torch.Generator(device="cuda").manual_seed(108)
        X8 = torch.randn(shape, generator=g, device="cuda").to(dt)
        inputs = {fname: X8, "fp16": X8.half(), "fp32": X8.float()}
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
        block = {}
        for k in inputs:
            cores = plans[k].run(inputs[k])
            prof[k].run(inputs[k])
            info = prof[k].info
            esize = inputs[k].element_size()
            gb, gf, pb, pf = step0_model(esize, vterms=2 if esize <= 2 else 3)
            gms, pms = info[8], info[10]
            block[k] = dict(
                call_gelem_s=dict(median=statistics.median(res[k]["call"]),
                                  spread=max(res[k]["call"]) - min(res[k]["call"]), runs=res[k]["call"]),
                batch_gelem_s=dict(median=statistics.median(res[k]["batch"]),
                                   spread=max(res[k]["batch"]) - min(res[k]["batch"]), runs=res[k]["batch"]),
                step0_gram_ms=gms, step0_factor_ms=pms, call_ms_profiled=info[4] + info[5] + info[6],
                step0_gram_model=dict(bytes=gb, flops=gf, tb_s=gb / gms / 1e9 if gms else None,
                                      tflop_s=gf / gms / 1e9 if gms else None),
                step0_proj_model=dict(bytes=pb, flops=pf, tb_s=pb / pms / 1e9 if pms else None,
                                      tflop_s=pf / pms / 1e9 if pms else None),
                speculative=int(plans[k].info[26]), kblocked_steps=int(plans[k].info[28]),
                rel_error_vs_f8=ops.tt_relative_error(X8, [c.clone() for c in cores]))
        out[fname] = block
        del inputs, plans, prof, bplans, batches, X8
        torch.cuda.empty_cache()
    with open(os.path.join(a.out, "bench_fp8.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
