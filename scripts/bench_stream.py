"""Dense TT-SVD of a tensor in host memory (ops.ttsvd_stream / tnb_ttsvd_stream) against the host-buffer call
(tnb_ttsvd_host: copy everything, then decompose) and the device-resident call (ops.ttsvd).

    python scripts/bench_stream.py --out DIR [--runs 3] [--big] [--noise-only]

In one run: the card's name and power limit; the host-to-device bandwidth from pinned memory, measured alone; 64^5 fp32
and bf16 at TT-rank 32 from pinned memory through the three calls, alternating, `runs` times: medians and spreads, the
effective input rate of the stream (2 x input bytes / time: step 0 reads the tensor twice) and its share of the measured
H2D rate.  With --big (when host RAM allows): one tensor larger than free device memory, 128^5 at TT-rank 16 (fp32, or
bf16 when RAM is short), built from a TT plus noise in pageable memory: its time, ranks and
ops.tt_relative_error_from_norm; what is skipped is printed with the reason.  --noise-only: the noise of a sum of chunk Grams (the streamed step 0's Gram) against the
fp64 Gram, ||G - (1 - c) G_64||_2 / ||G_64||_2 with c the least-squares shrink, for every tensor-core input type on the
three inputs of scripts/bench_fp16.py cut into 256 MiB chunks, beside the one-shot Gram's noise and the level the
accept rule allows for that type (ops.gram_noise_level).  Writes DIR/bench_stream.json (bench_stream_noise.json).
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


def stats(xs):
    return dict(median=statistics.median(xs), spread=max(xs) - min(xs), runs=xs)


def chunked_gram_noise():
    import torch

    from tntorch_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(11)
    mats = {"randn_16777216x64": lambda: torch.randn(1 << 24, 64, generator=g, device="cuda"),
            "randn_262144x2048": lambda: torch.randn(262144, 2048, generator=g, device="cuda"),
            "rank6_noise1e-3_16777216x64": lambda: (torch.randn(1 << 24, 6, generator=g, device="cuda")
                                                    @ torch.randn(6, 64, generator=g, device="cuda")
                                                    + 1e-3 * torch.randn(1 << 24, 64, generator=g, device="cuda"))}
    kinds = {"tf32": (torch.float32, lambda A: ops.gram(A, tensorcore=True)), "bf16": (torch.bfloat16, ops.gram_bf16),
             "fp16": (torch.float16, ops.gram_f16), "e4m3": (torch.float8_e4m3fn, ops.gram_f8),
             "e5m2": (torch.float8_e5m2, ops.gram_f8)}
    out = {}
    for name, make in mats.items():
        A32 = make()
        for kind, (dt, gram) in kinds.items():
            A = A32.to(dt)
            n = A.shape[1]
            rows = (256 << 20) // (n * A.element_size())  # the default chunk
            ref = torch.zeros(n, n, dtype=torch.float64, device="cuda")
            for i in range(0, A.shape[0], 1 << 20):
                B = A[i: i + (1 << 20)].double()
                ref += B.T @ B
            summed = torch.zeros_like(ref)
            for i in range(0, A.shape[0], rows):
                summed += gram(A[i: i + rows])
            nr = float(torch.linalg.matrix_norm(ref, ord=2))
            res = dict(chunks=-(-A.shape[0] // rows), level=ops.gram_noise_level(dt))
            for label, G in (("chunked", summed), ("one_shot", gram(A))):
                c = 1.0 - float((G * ref).sum() / (ref * ref).sum())
                res[label] = dict(bias_c=c, noise_rel_2norm=float(torch.linalg.matrix_norm(G - (1 - c) * ref, ord=2)) / nr)
            res["within_level"] = res["chunked"]["noise_rel_2norm"] <= res["level"]
            out[f"{name}/{kind}"] = res
            del A, ref, summed
        del A32
    return out


def h2d_gbs(nbytes=1 << 30, reps=10):
    import torch

    h = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    d = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    d.copy_(h, non_blocking=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        d.copy_(h, non_blocking=True)
    torch.cuda.synchronize()
    return reps * nbytes / (time.perf_counter() - t0) / 1e9


def host_ram_bytes():
    return os.sysconf("SC_PAGE_SIZE") * os.sysconf("SC_AVPHYS_PAGES")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--big", action="store_true")
    ap.add_argument("--noise-only", action="store_true")
    a = ap.parse_args()
    import torch

    from tntorch_b200 import ops

    os.makedirs(a.out, exist_ok=True)
    if a.noise_only:
        out = {"card": card(), "chunked_gram_noise": chunked_gram_noise()}
        with open(os.path.join(a.out, "bench_stream_noise.json"), "w") as f:
            json.dump(out, f, indent=1)
        print(json.dumps(out))
        return

    out = {"card": card(), "h2d_pinned_gb_s": h2d_gbs()}
    shape, r = [64] * 5, 32
    g = torch.Generator(device="cuda").manual_seed(108)
    for name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        Xd = torch.randn(shape, generator=g, device="cuda").to(dt)
        Xh = Xd.cpu().pin_memory()
        nbytes = Xd.numel() * Xd.element_size()
        dev_plan = ops.TTSVDPlan(shape, dt, rmax=r)
        host_plan = ops.TTSVDPlan(shape, dt, rmax=r, host_io=True)
        calls = {"stream": lambda: ops.ttsvd_stream(Xh, rmax=r), "host": lambda: host_plan.run_host(Xh),
                 "device": lambda: dev_plan.run(Xd)}
        for f in calls.values():  # warm-up
            f()
        torch.cuda.synchronize()
        times = {k: [] for k in calls}
        for _ in range(a.runs):
            for k, f in calls.items():  # alternating
                t0 = time.perf_counter()
                f()
                torch.cuda.synchronize()
                times[k].append(time.perf_counter() - t0)
        cores, info = ops.ttsvd_stream(Xh, rmax=r, return_info=True)
        ref = dev_plan.run(Xd)
        res = {k: stats([t * 1e3 for t in v]) for k, v in times.items()}
        rate = 2 * nbytes / statistics.median(times["stream"]) / 1e9
        res.update(input_gb=nbytes / 1e9, stream_input_rate_gb_s=rate, share_of_h2d=rate / out["h2d_pinned_gb_s"],
                   chunks=info["chunks"], passes=info["passes"], speculative=info["speculative"],
                   kblocked_steps=info["kblocked_steps"],
                   rel_error_stream=ops.tt_relative_error(Xd, cores), rel_error_device=ops.tt_relative_error(Xd, ref))
        out[f"64x5_r32_{name}"] = res
        del Xd, Xh, dev_plan, host_plan, cores, ref
        torch.cuda.empty_cache()

    if not a.big:
        out["big"] = "skipped: run with --big"
    else:
        free, _ = torch.cuda.mem_get_info()
        avail = host_ram_bytes()
        shape, r = [128] * 5, 16
        numel = 128 ** 5
        dt = torch.float32 if avail > 4 * numel * 1.2 else torch.bfloat16 if avail > 2 * numel * 1.3 else None
        if dt is None:
            out["big"] = f"skipped: {avail / 2**30:.0f} GiB of host RAM available, 128^5 needs 64 GiB in bf16"
        else:
            # a rank-16 TT plus 1e-2 noise, built slab by slab on the device into pageable host memory
            gg = torch.Generator(device="cuda").manual_seed(5)
            cores = [torch.randn(1 if k == 0 else r, 128, 1 if k == 4 else r, generator=gg, device="cuda") for k in range(5)]
            X = torch.empty(shape, dtype=dt)  # pageable: staged through the pinned pieces
            tail = torch.einsum("aib,bjc,ckd,dl->aijkl", cores[1], cores[2], cores[3], cores[4][:, :, 0]).reshape(r, -1)
            for i in range(128):
                slab = cores[0][0, i] @ tail
                slab = slab + 1e-2 * slab.std() * torch.randn(slab.shape, generator=gg, device="cuda")
                X[i].copy_(slab.reshape(shape[1:]).to(dt))
            del tail
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tc, info = ops.ttsvd_stream(X, rmax=r, return_info=True)
            torch.cuda.synchronize()
            t = time.perf_counter() - t0
            out["big"] = dict(shape=shape, dtype=str(dt), input_gb=X.numel() * X.element_size() / 1e9,
                              free_device_gb=free / 1e9, seconds=t, ranks=[1] + [int(c.shape[2]) for c in tc],
                              rel_error_from_norm=ops.tt_relative_error_from_norm(info["norm"], tc),
                              input_rate_gb_s=2 * X.numel() * X.element_size() / t / 1e9, chunks=info["chunks"],
                              passes=info["passes"], speculative=info["speculative"])
    with open(os.path.join(a.out, "bench_stream.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
